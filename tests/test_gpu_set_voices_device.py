"""`GpuBank.set_voices_device` (fdsp_bank_set_voices_device): `set_voices` with the values in device memory and the coefficients computed
on the device. It must leave a bank exactly where `set_voices` with the same values leaves it. So every case drives twin banks: H takes
`set_voices` with host values, D takes `set_voices_device` with the same values from device memory. Their rows must be bit for bit equal
after the call and after everything that follows it: more sets from either side, reset, clone, rate changes, grows, replace and crossfade
(all of which read the host graphs that D's device sets ran ahead of). On the CPU mock device (tests/test_set_voices_device_cpu.py) the
"device memory" is a host buffer."""
import ctypes as C
import os

import numpy as np
import pytest

from fundsp_b200 import workloads
from fundsp_b200.capi import ERR_ARG, ERR_UNSUPPORTED, FdspError
from fundsp_b200.net import Net
from fundsp_b200.prelude import *  # noqa: F401,F403
from fundsp_b200.sequencer import event, slot

pytestmark = pytest.mark.gpu
SR = 48000.0
MOCK = "mock" in os.environ.get("FDSP_B200_LIB", "")
V = 24
P_CENTER, P_CENTER_Q, P_CENTER_Q_GAIN, P_VALUE, P_BIQUAD, P_PAN = 1, 2, 3, 4, 6, 11
R = ((1, 1),)          # .right()


class HostBuf:
    """Values in the mock device's memory, which is host memory. The mock runs the bank's kernels when something synchronises, and host
    memory is not freed in stream order as a CUDA allocator frees it: every buffer stays alive until the test process ends."""
    KEEP = []

    def __init__(self, a):
        HostBuf.KEEP.append(self)
        self.a = np.ascontiguousarray(a, np.float32)
        self.__cuda_array_interface__ = {"shape": self.a.shape, "typestr": "<f4", "data": (self.a.ctypes.data, False), "strides": None,
                                         "version": 3}


def dev(vals):
    vals = np.ascontiguousarray(vals, np.float32)
    if MOCK:
        return HostBuf(vals)
    import torch
    return torch.from_numpy(vals).cuda()


def pair(voices, **kw):
    from fundsp_b200.bank import GpuBank
    return GpuBank(voices(), sample_rate=SR, per_voice=True, **kw), GpuBank(voices(), sample_rate=SR, per_voice=True, **kw)


def both(h, d, kind, vals, voices=None, address=()):
    """set_voices on H, set_voices_device on D."""
    vals = np.asarray(vals, np.float32).reshape(len(vals), -1)
    h.set_voices(kind, vals, voices=voices, address=address)
    d.set_voices_device(kind, dev(vals), voices=voices, address=address)


def same(h, d, n, what, finite=True):
    gh, gd = h.render_samples(n)[0], d.render_samples(n)[0]
    assert gh.shape == gd.shape, what
    if finite:
        assert np.isfinite(gh).all(), what
    bad = int((gh.view(np.uint32) != gd.view(np.uint32)).sum())
    assert bad == 0, (what, bad, np.nonzero((gh.view(np.uint32) != gd.view(np.uint32)).any(axis=(1, 2)))[0])
    return gh


def entries(rng, nvoices, n, values):
    vs = rng.integers(0, nvoices, n).astype(np.uint32)
    vs[: min(n, nvoices)] = rng.permutation(nvoices)[:n]   # every voice, then duplicates (the last one wins)
    return vs, np.asarray(values(rng, n), np.float32)


def _u(lo, hi, k=1):
    return lambda g, n: g.uniform(lo, hi, (n, k))


CQ = lambda g, n: np.stack([g.uniform(200, 5000, n), g.uniform(0.5, 8, n)], 1)                                   # noqa: E731
CQG = lambda g, n: np.stack([g.uniform(200, 5000, n), g.uniform(0.5, 8, n), g.uniform(0.25, 4, n)], 1)          # noqa: E731
BQ = lambda g, n: np.stack([-1.8 + 0.1 * g.uniform(0, 1, n), 0.82 + 0.05 * g.uniform(0, 1, n), 0.005 + 0.001 * g.uniform(0, 1, n),  # noqa: E731
                            np.full(n, 0.01), np.full(n, 0.005)], axis=1)
SVF = {"lowpass": lambda: lowpass_hz(1000.0, 1.0), "highpass": lambda: highpass_hz(800.0, 1.0), "bandpass": lambda: bandpass_hz(1500.0, 2.0),
       "notch": lambda: notch_hz(1200.0, 1.0), "peak": lambda: peak_hz(900.0, 1.5), "allpass": lambda: allpass_hz(700.0, 1.0),
       "bell": lambda: bell_hz(1000.0, 1.0, 2.0), "lowshelf": lambda: lowshelf_hz(600.0, 1.0, 0.5), "highshelf": lambda: highshelf_hz(3000.0, 0.7, 2.0)}


def saw_i(i):
    return saw_hz(110.0 + 7.0 * i)


def lp():
    return lowpass_hz(1000.0, 1.0)


# name: (voice i, kind, address, entry values (rng, n) -> [n, nvalues])
CASES = {f"svf_{m}_{k}": (lambda i, m=m: saw_i(i) >> SVF[m](), kind, R, vals)
         for m in SVF for k, kind, vals in (("center", P_CENTER, _u(200.0, 5000.0)), ("center_q", P_CENTER_Q, CQ), ("center_q_gain", P_CENTER_Q_GAIN, CQG))}
CASES.update({
    "butterpass": (lambda i: saw_i(i) >> butterpass_hz(900.0 + i), P_CENTER, R, _u(100.0, 8000.0)),
    "biquad": (lambda i: saw_i(i) >> biquad(-1.8, 0.82, 0.005, 0.01, 0.005), P_BIQUAD, R, BQ),
    "lowpole": (lambda i: saw_i(i) >> lowpole_hz(700.0 + i), P_CENTER, R, _u(50.0, 9000.0)),
    "highpole": (lambda i: saw_i(i) >> highpole_hz(300.0 + i), P_CENTER, R, _u(50.0, 9000.0)),
    "dcblock": (lambda i: saw_i(i) >> dcblock_hz(10.0 + i), P_CENTER, R, _u(1.0, 200.0)),
    "value_dc": (lambda i: (dc(110.0 + i) >> saw()) >> lp(), P_VALUE, ((1, 0), (1, 0)), _u(50.0, 900.0)),
    "value_dc_two_channels": (lambda i: dc((0.25 + 0.01 * i, -0.5)) >> (lp() | highpass_hz(300.0, 1.0)), P_VALUE, ((1, 0),), _u(-1.0, 1.0)),
    "pan": (lambda i: saw_i(i) >> pan(0.0), P_PAN, R, _u(-1.0, 1.0)),
    # entries that change nothing: a setting the node ignores, a center reaching the oscillator, an address that leads nowhere
    "pan_on_the_svf": (lambda i: saw_i(i) >> lp(), P_PAN, R, _u(-1.0, 1.0)),
    "center_on_the_oscillator": (lambda i: saw_i(i) >> lp(), P_CENTER, ((1, 0), (1, 1)), _u(200.0, 5000.0)),
    "address_leads_nowhere": (lambda i: saw_i(i) >> lp(), P_CENTER, ((1, 7),), _u(200.0, 5000.0)),
    # addresses through every combinator a setting walks
    "stack": (lambda i: (saw_i(i) >> lp()) | (saw_i(i + 1) >> highpass_hz(500.0, 1.0)), P_CENTER, ((1, 1), (1, 1)), _u(200.0, 5000.0)),
    "branch": (lambda i: saw_i(i) >> (lp() ^ highpass_hz(500.0, 1.0)), P_CENTER_Q, ((1, 1), (1, 0)), CQ),
    "bus": (lambda i: saw_i(i) >> (lp() & bandpass_hz(1500.0, 2.0)), P_CENTER, ((1, 1), (1, 1)), _u(200.0, 5000.0)),
    "binop": (lambda i: (saw_i(i) >> lp()) + (saw_i(i + 3) >> highpass_hz(800.0, 1.0)), P_CENTER, ((1, 0), (1, 1)), _u(200.0, 5000.0)),
    "unop": (lambda i: saw_i(i) >> (lp() * 0.5), P_CENTER, R, _u(200.0, 5000.0)),
    "thru": (lambda i: saw_i(i) >> thru(lp()), P_CENTER, R, _u(200.0, 5000.0)),
    "multi": (lambda i: saw_i(i) >> split(3) >> stacki(3, lambda k: lowpass_hz(600.0 + 300.0 * k, 1.0)), P_CENTER, ((1, 1), (1, 2)),
              _u(200.0, 5000.0)),
})


def twin_run(h, d, batch, mk, n=700):
    """The batch, then every operation after which H and D must still agree; `batch(h, d, rng)` applies one batch to both."""
    rng = np.random.default_rng(3)
    same(h, d, 300, "before")
    batch(h, d, rng)
    g = same(h, d, n, "after the batch")
    batch(h, d, rng)
    same(h, d, 64 * 3 + 5, "after a second batch")
    h.reset(); d.reset()
    same(h, d, n, "after reset")
    batch(h, d, rng)
    ch, cd = h.clone(), d.clone()
    same(ch, cd, n, "clones")
    same(h, d, n, "the originals after clone")
    for sr in (96000.0, 44100.0):
        batch(h, d, rng)
        h.set_sample_rate(sr); d.set_sample_rate(sr)
        same(h, d, n, ("after set_sample_rate", sr))
    batch(h, d, rng)
    h.add_voice(mk(V + 1)); d.add_voice(mk(V + 1))
    same(h, d, 333, "after add_voice")
    batch(h, d, rng)
    h.replace_voice(1, mk(V + 5)); d.replace_voice(1, mk(V + 5))
    same(h, d, 333, "after replace")
    batch(h, d, rng)
    # a voice moves to a class of its own (the setting passes a Unop unchanged), then a batch across both classes
    h.replace_voice(3, mk(V + 7) * 0.5); d.replace_voice(3, mk(V + 7) * 0.5)
    same(h, d, 333, "after a replace into another class")
    batch(h, d, rng)
    same(h, d, 333, "a batch after the replace into another class")
    h.crossfade_voice(2, 1, 0.005, mk(V + 6)); d.crossfade_voice(2, 1, 0.005, mk(V + 6))
    same(h, d, 700, "after crossfade")
    batch(h, d, rng, skip=2)   # (the crossfading vertex takes no device set)
    same(h, d, 700, "a batch after the crossfade")
    return g


@pytest.mark.parametrize("name", sorted(CASES))
def test_device_batch_equals_the_host_batch(name):
    mk, kind, addr, values = CASES[name]
    h, d = pair(lambda: [mk(i) for i in range(V)])

    def batch(h, d, rng, skip=None):
        vs, vals = entries(rng, h.voices(), 2 * V + 5, values)
        keep = vs != skip
        both(h, d, kind, vals[keep], vs[keep], addr)

    g = twin_run(h, d, batch, mk)
    assert np.abs(g).max() > 1e-4
    # sets from the host after the device's: they must start from what the device left (the host graphs were reconciled)
    vs, vals = entries(np.random.default_rng(9), 4, 4, values)
    for b in (h, d):
        b.set(0, kind, tuple(float(x) for x in vals[0]), address=addr)
        b.set_voices(kind, vals[1:], voices=vs[1:], address=addr)
    same(h, d, 200, "after host sets")


def test_two_addresses_that_reach_one_node():
    """A Unop passes a setting on without peeling it, so (.right()) and (.right(), .left()) both reach the filter of saw >> lp() * 0.5: the
    device's sets through either address start from what the other left."""
    h, d = pair(lambda: [saw_i(i) >> (lp() * 0.5) for i in range(V)])
    k1, k2 = R, ((1, 1), (1, 0))
    rng = np.random.default_rng(8)
    same(h, d, 100, "before")
    both(h, d, P_CENTER_Q, CQ(rng, V), None, k2)
    same(h, d, 300, "center_q through the longer address")
    both(h, d, P_CENTER, _u(200.0, 5000.0)(rng, V), None, k1)
    same(h, d, 300, "center through the shorter address")
    both(h, d, P_CENTER_Q, CQ(rng, V // 2), np.arange(0, V, 2, dtype=np.uint32), k1)
    both(h, d, P_CENTER, _u(200.0, 5000.0)(rng, V), None, k2)
    same(h, d, 300, "both again")
    h.reset(); d.reset()
    same(h, d, 600, "after reset (the host graphs)")
    same(h.clone(), d.clone(), 300, "clones")


def test_nodes_that_differ_under_one_class_signature():
    """dc and var lower alike (Constant<1>), as do biquad, butterpass and resonator (Biquad): one class, different nodes per voice. Each
    voice's node is checked on its own: a target takes the set, a node that ignores the setting is skipped, any other is refused with the
    entry's index before anything is applied."""
    from fundsp_b200.bank import GpuBank
    from fundsp_b200.shared import shared
    mk = [lambda i: dc(400.0 + i) >> sine(), lambda i: var(260.0 + 2.0 * i) >> sine(), lambda i: dc(500.0 + 3.0 * i) >> sine(), lambda i: var(250.0 + i) >> sine()]
    voices = lambda: [mk[(i * 3) % 4](i) for i in range(4 * 4)]   # noqa: E731   (the first voice a var)
    h, d = GpuBank(voices(), sample_rate=SR, per_voice=True), GpuBank(voices(), sample_rate=SR, per_voice=True)
    assert len(d.classes()) == 1
    same(h, d, 100, "before")
    consts = np.array([i for i in range(16) if (i * 3) % 4 in (0, 2)], np.uint32)
    vars_ = np.array([i for i in range(16) if (i * 3) % 4 in (1, 3)], np.uint32)
    both(h, d, P_VALUE, np.linspace(200.0, 900.0, len(consts)), consts, ((1, 0),))
    same(h, d, 600, "value on the dc voices")
    vals = np.full((3, 1), 700.0, np.float32)
    l0 = d.launch_count()
    with pytest.raises(FdspError) as e:
        d.set_voices_device(P_VALUE, dev(vals), voices=np.array([consts[0], consts[1], vars_[0]], np.uint32), address=((1, 0),))
    assert e.value.code == ERR_UNSUPPORTED and e.value.entry == 2 and d.launch_count() == l0, str(e.value)
    same(h, d, 300, "after the refusal")
    both(h, d, P_PAN, np.zeros(16), None, ((1, 0),))   # every node there ignores pan
    same(h, d, 300, "an ignored setting")
    h.reset(); d.reset()
    same(h, d, 300, "after reset")
    # a var(&shared) voice makes that row a Shared reader row, which the bank rewrites whole from the host: refused, nothing applied
    sh = shared(300.0)
    voices = lambda: [var(sh) >> sine()] + [dc(400.0 + i) >> sine() for i in range(1, 6)]   # noqa: E731
    h, d = GpuBank(voices(), sample_rate=SR, per_voice=True), GpuBank(voices(), sample_rate=SR, per_voice=True)
    assert len(d.classes()) == 1
    with pytest.raises(FdspError) as e:
        d.set_voices_device(P_VALUE, dev(np.full((2, 1), 700.0)), voices=np.array([4, 0], np.uint32), address=((1, 0),))
    assert e.value.code == ERR_UNSUPPORTED and e.value.entry == 0, str(e.value)
    same(h, d, 300, "Shared reader row refused")

    kinds = [lambda i: saw_i(i) >> biquad(-1.8, 0.82, 0.005, 0.01, 0.005), lambda i: saw_i(i) >> butterpass_hz(900.0 + i),
             lambda i: saw_i(i) >> resonator_hz(800.0 + i, 50.0)]
    voices = lambda: [kinds[(i * 5) % 3](i) for i in range(12)]   # noqa: E731
    h, d = GpuBank(voices(), sample_rate=SR, per_voice=True), GpuBank(voices(), sample_rate=SR, per_voice=True)
    assert len(d.classes()) == 1
    same(h, d, 100, "biquads before")
    of = lambda k: np.array([i for i in range(12) if (i * 5) % 3 == k], np.uint32)   # noqa: E731
    rng = np.random.default_rng(12)
    both(h, d, P_BIQUAD, BQ(rng, len(of(0))), of(0), R)
    both(h, d, P_CENTER, _u(300.0, 3000.0)(rng, len(of(1))), of(1), R)
    both(h, d, P_BIQUAD, BQ(rng, 12), None, R)   # butterpass and resonator ignore biquad
    same(h, d, 600, "biquad on the biquads, center on the butterpasses")
    with pytest.raises(FdspError) as e:   # the resonator's host set takes center
        d.set_voices_device(P_CENTER, dev(np.full((2, 1), 900.0)), voices=np.array([of(1)[0], of(2)[0]], np.uint32), address=R)
    assert e.value.code == ERR_UNSUPPORTED and e.value.entry == 1, str(e.value)
    same(h, d, 300, "after the refusal")
    same(h.clone(), d.clone(), 300, "clones")


def test_set_leaves_state_and_reset_image_alone():
    """What the device path assumes: each target's set changes its parameter words only (checked on the host lowering)."""
    from fundsp_b200 import capi
    L = capi.lib()
    nodes = [(f(), P_CENTER_Q_GAIN, (700.0, 3.0, 0.5)) for f in SVF.values()] + [
        (butterpass_hz(500.0), P_CENTER, (2000.0,)), (biquad(-1.7, 0.8, 0.01, 0.02, 0.01), P_BIQUAD, (-1.5, 0.6, 0.1, 0.2, 0.1)),
        (lowpole_hz(300.0), P_CENTER, (900.0,)), (highpole_hz(300.0), P_CENTER, (900.0,)), (dcblock_hz(20.0), P_CENTER, (40.0,)),
        (dc((1.0, 2.0, 3.0)), P_VALUE, (0.5,)), (pan(0.2), P_PAN, (-0.7,))]
    for node, kind, vals in nodes:
        hd = capi.NodeHandle(node)
        P0, S0, U0 = hd.lowering()
        capi.check(L.fdsp_node_set(hd.h, kind, (C.c_float * 5)(*vals), len(vals), 0, (C.c_int64 * 1)(0), 0))
        P1, S1, U1 = hd.lowering()
        assert np.array_equal(S0, S1) and np.array_equal(U0, U1) and not np.array_equal(P0, P1), hd.signature()


EDGES = {
    "cutoff": [0.0, -300.0, 24000.0, 30000.0, 1.0e7, 3.0e30, np.nan, np.inf, -np.inf, 1.0e-30],
    "q": [1.0e-30, 1.0e-6, 0.0, -1.0, np.nan, np.inf],
    "gain": [0.0, -1.0, 1.0e-30, np.inf, np.nan],
}


@pytest.mark.parametrize("mode", sorted(SVF))
def test_control_edges(mode):
    """Cutoffs at 0, negative, at and past Nyquist, large enough for the large-argument tanf reduction, non-finite; q near 0; gain 0:
    whatever the host lowering of the same value gives."""
    h, d = pair(lambda: [saw_i(i) >> SVF[mode]() for i in range(V)])
    cut = EDGES["cutoff"]
    rows = [(c, 1.0, 1.0) for c in cut] + [(1000.0, q, 1.0) for q in EDGES["q"]] + [(1000.0, 1.0, g) for g in EDGES["gain"]]
    vals = np.array(rows[:V] + [(500.0 + 10 * i, 1.0, 1.0) for i in range(V - len(rows))], np.float32)
    both(h, d, P_CENTER_Q_GAIN, vals, None, R)
    same(h, d, 200, "edges", finite=False)
    both(h, d, P_CENTER, np.array(cut * 3, np.float32)[:V], np.arange(V, dtype=np.uint32)[::-1].copy(), R)
    same(h, d, 200, "edge cutoffs", finite=False)
    for k in range(V):
        for b in (h, d):
            b.set(k, P_CENTER_Q_GAIN, (800.0, 1.0, 1.0), address=R)
    same(h, d, 300, "back to finite controls", finite=False)   # (a non-finite filter state stays until reset)
    h.reset(); d.reset()
    same(h, d, 300, "after reset")


def test_partial_settings_after_full_ones():
    """center after center_q_gain from the device keeps q and gain; host sets then start from the device's controls."""
    h, d = pair(lambda: [saw_i(i) >> bell_hz(1000.0, 1.0, 2.0) for i in range(V)])
    rng = np.random.default_rng(4)
    both(h, d, P_CENTER_Q_GAIN, CQG(rng, V), None, R)
    both(h, d, P_CENTER, _u(200.0, 5000.0)(rng, V), None, R)
    same(h, d, 300, "center after center_q_gain")
    both(h, d, P_CENTER_Q, CQ(rng, V // 2), np.arange(0, V, 2, dtype=np.uint32), R)
    for b in (h, d):
        b.set(3, P_CENTER, (1234.0,), address=R)
        b.set_voices(P_CENTER, np.full((3, 1), 2345.0, np.float32), voices=np.array([4, 6, 8], np.uint32), address=R)
    same(h, d, 300, "host sets after device sets")
    both(h, d, P_CENTER, np.full((V, 1), 800.0, np.float32), None, R)
    same(h, d, 300, "device center after host sets")


MIXED = [lambda i: saw_i(i) >> lp(), lambda i: noise().seed(i) >> lp(), lambda i: (dc(110.0 + i) >> sine()) >> lp()]


def test_classes_interleaved_duplicates_and_empty():
    kinds = [(i * 7) % 3 for i in range(3 * V)]
    h, d = pair(lambda: [MIXED[k](i) for i, k in enumerate(kinds)])
    assert len(d.classes()) == 3
    same(h, d, 200, "before")
    rng = np.random.default_rng(5)
    for n in (1, 2, 64, 3 * V, 5 * V):
        vs, vals = entries(rng, 3 * V, n, _u(200.0, 5000.0))
        l0 = d.launch_count()
        both(h, d, P_CENTER, vals, vs, R)
        assert d.launch_count() - l0 == len({kinds[v] for v in vs}), n
        same(h, d, 129, ("after", n))
    vals = np.linspace(300.0, 3000.0, 3 * V, dtype=np.float32)
    both(h, d, P_CENTER, vals.reshape(-1, 1), None, R)
    same(h, d, 200, "voices=None")
    l0 = d.launch_count()
    d.set_voices_device(P_CENTER, dev(np.zeros((0, 1), np.float32)), address=R)
    assert d.launch_count() == l0
    same(h, d, 200, "empty batch")


def test_sequencer_events():
    mk = lambda i: event(saw_i(i) >> lp(), (30.0 + 97.3 * i) / SR, (30.0 + 97.3 * i + (400.0 if i % 3 == 0 else 9000.0)) / SR, i % 2,  # noqa: E731
                         40.0 / SR, 100.0 / SR)
    h, d = pair(lambda: [mk(i) for i in range(V)], mix=True)
    rng = np.random.default_rng(6)
    same(h, d, 100, "before")
    for k in range(3):
        vs, vals = entries(rng, h.voices(), V + 7, CQ)
        both(h, d, P_CENTER_Q, vals, vs, R)
        same(h, d, 600, ("batch", k))
    h.push_event(mk(V + 3)); d.push_event(mk(V + 3))
    same(h, d, 300, "after push_event")
    vs, vals = entries(rng, h.voices(), V + 7, CQ)
    both(h, d, P_CENTER_Q, vals, vs, R)
    same(h, d, 600, "batch after push_event")
    h.reset(); d.reset()
    same(h, d, 600, "after reset")


def test_refusals_apply_nothing():
    """Every refusal: its code and entry, no launch, and a bank (and its clone, built from its host graphs) equal to an untouched twin."""
    from fundsp_b200.bank import GpuBank
    mk = [lambda i: saw_i(i) >> lp(),
          lambda i: slot(saw_i(i) >> lp()),
          lambda i: update(saw_i(i) >> lp(), 0.004, "|t, dt, x| x.set(Setting::center(600.0 + 400.0 * sin_hz(r, t)).right())", r=1.0 + 0.1 * i),
          lambda i: saw_i(i) >> moog_hz(1000.0, 0.5),
          lambda i: saw_i(i) >> lowrez_hz(1000.0, 0.5),
          lambda i: saw_i(i) >> resonator_hz(1000.0, 100.0)]
    voices = lambda: [mk[i % len(mk)](i) for i in range(2 * len(mk))]   # noqa: E731
    t, d = GpuBank(voices(), sample_rate=SR, per_voice=True), GpuBank(voices(), sample_rate=SR, per_voice=True)
    same(t, d, 100, "before")
    vals = np.linspace(300.0, 2000.0, 8, dtype=np.float32).reshape(-1, 1)
    cases = [(np.array([0, 6, 12, 0, 0, 0, 0, 0], np.uint32), ERR_ARG, 2, R),     # out of range
             (np.array([0, 6, 7, 0, 0, 0, 0, 0], np.uint32), ERR_UNSUPPORTED, 2, R),   # a Slot voice
             (np.array([6, 0, 6, 8, 0, 0, 0, 0], np.uint32), ERR_UNSUPPORTED, 3, R),   # update(): a System
             (np.array([0, 9, 0, 0, 0, 0, 0, 0], np.uint32), ERR_UNSUPPORTED, 1, R),   # the Moog
             (np.array([0, 0, 0, 0, 0, 0, 10, 0], np.uint32), ERR_UNSUPPORTED, 6, R),  # Rez
             (np.array([0, 0, 5, 0, 0, 0, 0, 0], np.uint32), ERR_UNSUPPORTED, 2, R),   # a fixed Resonator (its host set changes it)
             (np.array([0, 6, 0, 0, 0, 0, 0, 0], np.uint32), ERR_UNSUPPORTED, 0, ((2, 5),))]   # .node(id)
    for vs, code, entry, addr in cases:
        l0 = d.launch_count()
        with pytest.raises(FdspError) as e:
            d.set_voices_device(P_CENTER, dev(vals), voices=vs, address=addr)
        assert e.value.code == code and e.value.entry == entry, (vs, e.value.code, e.value.entry, str(e.value))
        assert d.launch_count() == l0
    same(t, d, 500, "after the refusals")
    same(t.clone(), d.clone(), 300, "clones after the refusals")
    # a crossfading vertex of a Net bank
    net_mk = lambda i: noise().seed(i) >> lowpass_hz(300.0 + 100.0 * i, 1.0) >> pan(0.0)   # noqa: E731

    def net():
        n = Net.wrap(net_mk(0))
        for i in range(1, 6):
            n = n & Net.wrap(net_mk(i))
        return n
    t, d = GpuBank.from_net(net(), per_voice=True, sample_rate=SR), GpuBank.from_net(net(), per_voice=True, sample_rate=SR)
    for b in (t, d):
        b.crossfade_voice(2, 1, 0.01, net_mk(40))
    with pytest.raises(FdspError) as e:
        d.set_voices_device(P_CENTER_Q, dev(np.ones((3, 2), np.float32) * 700.0), voices=np.array([0, 1, 2], np.uint32), address=((1, 0), (1, 1)))
    assert e.value.code == ERR_UNSUPPORTED and e.value.entry == 2
    same(t, d, 500, "crossfading vertex refused")


def test_stream_order():
    """A side stream writes the values, the call runs, then the same stream overwrites them: the bank has the first values."""
    if MOCK:
        pytest.skip("the mock device's values are host memory written by the host")
    import torch
    h, d = pair(lambda: [saw_i(i) >> lp() for i in range(V)])
    same(h, d, 100, "before")
    first = np.linspace(300.0, 3000.0, V, dtype=np.float32).reshape(-1, 1)
    buf = torch.zeros((V, 1), dtype=torch.float32, device="cuda")
    src = torch.from_numpy(first).cuda()
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)   # the values land long after the call returns
        buf.copy_(src)
        d.set_voices_device(P_CENTER, buf, address=R)
        buf.fill_(99.0)
    h.set_voices(P_CENTER, first, address=R)
    same(h, d, 400, "first values")
    torch.cuda.synchronize()


# what the device is given, read from a CUDA trace (torch.profiler, in a process of its own): per batch one scatter kernel per class
# touched and one host-to-device copy, of the entry indices (8 bytes an entry; the values would be 12), and no device-to-host copy but
# each process() output
TRACE = '''
import json, sys, tempfile, numpy as np, torch
from torch.profiler import ProfilerActivity, profile
from fundsp_b200.bank import GpuBank
from fundsp_b200.prelude import bell_hz, noise, saw_hz
mk = [lambda i: saw_hz(110.0 + 7.0 * i) >> bell_hz(1000.0, 1.0, 2.0), lambda i: noise().seed(i) >> bell_hz(1000.0, 1.0, 2.0)]
V = 2000
b = GpuBank([mk[i % 2](i) for i in range(V)], per_voice=False, mix=True, sample_rate=48000.0)
vals = torch.rand((V, 3), device="cuda") * torch.tensor([3000.0, 4.0, 2.0], device="cuda") + torch.tensor([200.0, 0.5, 0.25], device="cuda")
vs = (np.arange(V) * 7 % V).astype(np.uint32)
for k in range(3):
    b.set_voices_device(3, vals, voices=vs, address=((1, 1),)); b.process(64)
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as p:
    for k in range(100):
        vals.mul_(0.999)
        b.set_voices_device(3, vals, voices=vs, address=((1, 1),))
        b.process(64)
    torch.cuda.synchronize()
f = tempfile.mktemp(suffix=".json")
p.export_chrome_trace(f)
ev = [e for e in json.load(open(f))["traceEvents"] if e.get("ph") == "X"]
h2d = [e["args"].get("bytes") for e in ev if "Memcpy HtoD" in e.get("name", "")]
d2h = [e for e in ev if "Memcpy DtoH" in e.get("name", "")]
scat = [e for e in ev if "set_controls_kernel" in e.get("name", "")]
print("trace", len(h2d), sorted(set(h2d)), len(d2h), len(scat), flush=True)
'''


def test_trace_one_scatter_per_class_and_no_copy_of_the_values():
    if MOCK:
        pytest.skip("a CUDA trace needs the GPU (the launch counts are checked above on the mock device too)")
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", TRACE], capture_output=True, text=True, cwd=root, timeout=900, env=dict(os.environ, PYTHONPATH=root))
    lines = [ln.split(maxsplit=1)[1] for ln in r.stdout.splitlines() if ln.startswith("trace ")]
    assert r.returncode == 0 and len(lines) == 1, (r.stdout[-1500:], r.stderr[-1500:])
    n_h2d, sizes, n_d2h, n_scat = _parse(lines[0])
    assert n_scat == 2 * 100, lines[0]
    assert n_h2d == 100 and sizes == [8 * 2000], lines[0]
    assert n_d2h <= 100, lines[0]


def _parse(s):
    a, rest = s.split(" ", 1)
    sizes, rest = rest.split("]", 1)
    b, c = rest.split()
    return int(a), [int(x) for x in sizes.strip("[ ").split(",") if x.strip()], int(b), int(c)


# ---- the headline bank: every voice's cutoff and q from a GPU-computed tensor before every call
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
        got = []
        for k, n in enumerate(calls):
            if MOCK:
                rng = np.random.default_rng(17 + k)
                cq = np.stack([rng.uniform(200, 8000, nv), rng.uniform(0.5, 8, nv)], 1).astype(np.float32)
                vals = HostBuf(cq)
            else:
                import torch
                g = torch.Generator(device="cuda").manual_seed(17 + k)
                vals = torch.rand((nv, 2), device="cuda", generator=g) * torch.tensor([7800.0, 7.5], device="cuda") + torch.tensor([200.0, 0.5], device="cuda")
                cq = vals.cpu().numpy()
            for bank in (bm, bv):
                bank.set_voices_device(P_CENTER_Q, vals, address=R)
            if n > 64:
                rows, _ = bv.render_samples(n)
                _, mix = bm.render_samples(n)
                segs = launch_segments(n, classes, nv, 1, False, False)
            else:
                rows = bv.process(n).reshape(nv, 1, n)
                mix = bm.process(n)
                segs = [(0, n)]
            check_mix(mix, rows, classes, segs, False, (rt, k, n))
            got.append((rows, mix, cq))
        outs[rt] = got
    for (r1, m1, _), (r0, m0, _) in zip(outs["1"], outs["0"]):
        assert np.array_equal(r1, r0) and np.array_equal(m1, m0), "FDSP_RT=1 and FDSP_RT=0 differ"
    pick = range(nv) if MOCK else sorted(set(range(0, nv, 97)) | {nv - 1})
    for v in pick:
        u = OracleUnit(workloads.saw_svf_voice(v)); u.set_sample_rate(SR)
        for (rows, _, cq), n in zip(outs["1"], calls):
            u.L.fo_set(u.h, P_CENTER_Q, (C.c_float * 2)(*cq[v]), 2, 0, (C.c_int64 * 2)(1, 1), 1)
            want = u.process_many(n) if n > 64 else u.process(n)
            assert np.array_equal(rows[v], want.reshape(rows[v].shape)), (v, n, int((rows[v] != want.reshape(rows[v].shape)).sum()))

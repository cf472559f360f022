"""Shared controls on the GPU: var(s) readers that follow Shared.set between calls, monitor(s, meter) and timer(s) writers whose values are
stored back after every call. Each case drives oracle units (oracle/fo_shared.h, over oracle cells of their own) with the same sets at
the same call boundaries and compares every voice bit for bit, and every written Shared exactly."""
import os
import threading

import numpy as np
import pytest

from fundsp_b200.bank import GpuBank
from fundsp_b200.capi import FdspError
from fundsp_b200.net import Net
from fundsp_b200.prelude import *  # noqa: F401,F403
from fundsp_b200.sequencer import event, slot
from oracle import OracleUnit, lib as olib
from oracle_shared import mirror, set_both
from test_gpu_mix import MOCK, bank_classes, check_mix, launch_segments, mix_model

pytestmark = pytest.mark.gpu
SR = 48000.0
BIG = 512 if MOCK else 16384


def units(voices):
    olib().fo_set_denormal_emulation(0)
    us = [OracleUnit(v) for v in voices]
    for u in us:
        u.set_sample_rate(SR)
    return us


def oracle_rows(us, n):
    return np.stack([u.process_many(n) for u in us])


def saw_voice(s, i):
    return var(s) * saw_hz(110.0 + (i % 97) * 3.0) >> lowpass_hz(500.0 + (i % 13) * 100.0, 0.7 + (i % 5) * 0.1)


def test_two_shareds_many_voices_ragged_process_and_render():
    a, b = shared(0.5), shared(-0.25)
    mk = lambda i: saw_voice(a if i % 3 else b, i)
    bank = GpuBank([mk(i) for i in range(BIG)], per_voice=True, mix=True, sample_rate=SR)
    us = units([mk(i) for i in range(BIG)])
    classes = bank_classes(bank, [mk(i) for i in range(BIG)])
    for size, va, vb in ((64, None, None), (17, 0.75, None), (1, None, 2.0), (33, -1.0, -1.0), (64, None, None), (5, 0.125, 0.0)):
        if va is not None:
            set_both(a, va)
        if vb is not None:
            set_both(b, vb)
        got = bank.process(size)
        want = mix_model(oracle_rows(us, size), classes, [(0, size)], False)
        assert np.array_equal(got, want), (size, float(np.abs(got - want).max()))
    for n, va, vb in ((1000, 0.3, None), (777, None, 0.9), (2048 + 5, -0.5, 0.25)):
        if va is not None:
            set_both(a, va)
        if vb is not None:
            set_both(b, vb)
        rows, mix = bank.render_samples(n)
        want = oracle_rows(us, n)
        assert np.array_equal(rows, want), (n, int((rows != want).sum()))
        check_mix(mix, rows, classes, launch_segments(n, classes, BIG, 1, True, False), False, "render")


def test_keys_pattern_var_follow_drives_a_cutoff():
    cut = shared(800.0)   # examples/keys.rs:171-178: var(&s) >> follow(0.01)
    mk = lambda i: (saw_hz(55.0 + 11.0 * i) | var(cut) >> follow(0.01) | dc(1.0)) >> lowpass()
    bank = GpuBank([mk(i) for i in range(24)], per_voice=True, sample_rate=SR)
    us = units([mk(i) for i in range(24)])
    for n, v in ((700, None), (1300, 3000.0), (64, 120.0), (2500, 1500.0)):
        if v is not None:
            set_both(cut, v)
        rows, _ = bank.render_samples(n)
        assert np.array_equal(rows, oracle_rows(us, n)), n


METERS = (Meter.Sample, Meter.Peak(0.02), Meter.Rms(0.05))


@pytest.mark.parametrize("k", range(3))
def test_monitor_and_timer_write_back_last_writer_wins(k):
    m_own = [shared(7.0) for _ in range(4)]
    m_all, t = shared(9.0), shared(5.0)
    mk = lambda i: ((noise().seed(i) * (0.2 + 0.1 * i) >> monitor(m_own[i % 4], METERS[k]) >> monitor(m_all, METERS[(k + i) % 3])
                     >> lowpass_hz(900.0 + 50 * i, 1.0)) | timer(t))
    bank = GpuBank([mk(i) for i in range(11)], per_voice=True, mix=True, sample_rate=SR)
    assert t.value() == 0.0   # Timer::new stores 0
    us = units([mk(i) for i in range(11)])
    for size in (64, 13, 1, 64, 40, 7, 64):
        bank.process(size)
        for u in us:
            u.process_many(size)
        for s in m_own + [m_all, t]:
            assert s.value() == mirror(s).value(), (size, s.value(), mirror(s).value())
    for n in (1000, 4097):
        rows, _ = bank.render_samples(n)
        assert np.array_equal(rows, oracle_rows(us, n))
        for s in m_own + [m_all, t]:
            assert s.value() == mirror(s).value(), (n, s.value(), mirror(s).value())
    assert t.value() > 0.0 and m_all.value() != 9.0


def test_timer_known_answer_and_reset_and_rate_change():
    t = shared(1.0)
    bank = GpuBank([timer(t) | dc(0.0)], per_voice=True, sample_rate=SR)
    us = units([timer(t) | dc(0.0)])
    for _ in range(5):
        bank.process(64)
    exact = np.float64(0.0)
    for _ in range(5):
        exact += 64.0 * (1.0 / SR)
    assert t.value() == float(np.float32(exact))
    bank.reset()
    us[0].reset()
    assert t.value() == 0.0
    bank.set_sample_rate(44100.0)
    us[0].set_sample_rate(44100.0)
    for n in (100, 64, 3):
        bank.render_samples(n)
        us[0].process_many(n)
    assert t.value() == mirror(t).value()


def test_one_shared_read_by_two_banks_and_a_clone():
    s = shared(0.3)
    mk = lambda i: saw_voice(s, i)
    b1 = GpuBank([mk(i) for i in range(8)], per_voice=True, sample_rate=SR)
    b2 = GpuBank([mk(i) for i in range(8, 20)], per_voice=True, sample_rate=SR)
    u1, u2 = units([mk(i) for i in range(8)]), units([mk(i) for i in range(8, 20)])
    r1, _ = b1.render_samples(500)
    oracle_rows(u1, 500)
    b3 = b1.clone()
    u3 = units([mk(i) for i in range(8)])
    oracle_rows(u3, 500)
    for n, v in ((300, 0.9), (129, -0.6)):
        set_both(s, v)
        for b, us in ((b1, u1), (b2, u2), (b3, u3)):
            rows, _ = b.render_samples(n)
            assert np.array_equal(rows, oracle_rows(us, n)), n


def test_readers_inside_a_net_an_event_and_a_slot():
    s = shared(0.4)
    net_voice = lambda i: ((Net.wrap(var(s)) | Net.wrap(saw_hz(100.0 + i))) >> Net.wrap(pass_() * pass_())).node()
    ev = lambda i: event(var(s) * saw_hz(200.0 + i), (10.0 + 30.0 * i) / SR, (2000.0 + 30.0 * i) / SR, 1, 40.0 / SR, 100.0 / SR)
    sl = lambda i: slot(var(s) * noise().seed(i))
    for mk in (net_voice, ev, sl):
        bank = GpuBank([mk(i) for i in range(6)], per_voice=True, sample_rate=SR)
        us = units([mk(i) for i in range(6)])
        for n, v in ((400, None), (333, 0.8), (1500, -0.2)):
            if v is not None:
                set_both(s, v)
            rows, _ = bank.render_samples(n)
            assert np.array_equal(rows, oracle_rows(us, n)), (mk, n)


def test_a_setter_thread_joined_before_each_call():
    s = shared(0.0)
    mk = lambda i: saw_voice(s, i)
    bank = GpuBank([mk(i) for i in range(16)], per_voice=True, sample_rate=SR)
    us = units([mk(i) for i in range(16)])
    for k in range(5):
        th = threading.Thread(target=lambda k=k: [s.set(0.1 * k + 0.01 * j) for j in range(100)])
        th.start()
        th.join()
        mirror(s).set(s.value())
        rows, _ = bank.render_samples(257)
        assert np.array_equal(rows, oracle_rows(us, 257)), k


def test_resident_kernel_on_and_off_give_the_same_bits():
    """A Shared bank declines the resident process() kernel (one launch per call, also with FDSP_RT=1), while the same bank with var(0.5)
    takes it; both settings give the same bits."""
    s = shared(0.5)
    mk = lambda i, x: saw_voice(x, i)
    outs, launches = [], []
    for rt in ("1", "0"):
        os.environ["FDSP_RT"] = rt
        try:
            s.set(0.5)
            bank = GpuBank([mk(i, s) for i in range(64)], per_voice=False, mix=True, sample_rate=SR)
            got, l0 = [], bank.launch_count()
            for k in range(12):
                if k % 4 == 3:
                    s.set(0.1 * k)
                got.append(bank.process(64 if k % 5 else 31))
            outs.append(np.concatenate(got, axis=1))
            launches.append(bank.launch_count() - l0)
            del bank
        finally:
            os.environ.pop("FDSP_RT", None)
    assert np.array_equal(outs[0], outs[1])
    assert launches[0] >= 12 and launches[0] == launches[1], launches   # a launch per call on both settings
    if not MOCK:                                                          # (the mock device has no resident kernel)
        os.environ["FDSP_RT"] = "1"
        try:
            plain = GpuBank([mk(i, 0.5) for i in range(64)], per_voice=False, mix=True, sample_rate=SR)
            l0 = plain.launch_count()
            for k in range(12):
                plain.process(64)
            assert plain.launch_count() - l0 < 12   # this one is served by the resident kernel
            del plain
        finally:
            os.environ.pop("FDSP_RT", None)


def test_var_fn_with_a_tuple_result():
    s = shared(0.25)
    mk = lambda i: (var_fn(s, "|x| { let y = x * g; (y, tanh(y) - x.abs().sqrt()) }", 2, g=1.0 + 0.1 * i) | saw_hz(90.0 + i)) >> (
        pass_() * pass_() | pass_())
    bank = GpuBank([mk(i) for i in range(20)], per_voice=True, sample_rate=SR)
    assert len(bank.classes()) == 1
    us = units([mk(i) for i in range(20)])
    for size, v in ((64, None), (23, 0.9), (1, -0.5)):
        if v is not None:
            set_both(s, v)
        bank.process(size)
        for u in us:
            u.process_many(size)
    for n, v in ((700, 2.0), (1333, -0.125)):
        set_both(s, v)
        rows, _ = bank.render_samples(n)
        assert np.array_equal(rows, oracle_rows(us, n)), n


def test_rate_change_and_reset_with_readers_and_writers_running():
    a, m, t = shared(0.7), shared(0.0), shared(0.0)
    mk = lambda i: ((var(a) * saw_hz(150.0 + 7 * i) >> monitor(m, Meter.Rms(0.01)) >> lowpass_hz(800.0, 1.0)) | timer(t))
    bank = GpuBank([mk(i) for i in range(9)], per_voice=True, sample_rate=SR)
    us = units([mk(i) for i in range(9)])

    def step(n, v=None):
        if v is not None:
            set_both(a, v)
        rows, _ = bank.render_samples(n)
        assert np.array_equal(rows, oracle_rows(us, n)), n
        for s in (m, t):
            assert s.value() == mirror(s).value(), (n, s.value(), mirror(s).value())

    step(1000)
    step(333, 0.2)
    bank.set_sample_rate(44100.0)   # the timer keeps its time; the readers and monitor follow the new rate
    for u in us:
        u.set_sample_rate(44100.0)
    step(777, -0.4)
    bank.reset()
    for u in us:
        u.reset()
    assert t.value() == 0.0 and mirror(t).value() == 0.0
    step(500)
    step(64, 1.5)


def test_refusals_name_the_shared():
    s = shared(0.0)
    with pytest.raises(FdspError, match="Shared at .* both read .* and written"):
        GpuBank([var(s) >> monitor(s, Meter.Sample), dc(0.0) >> monitor(shared(), Meter.Sample)], sample_rate=SR)
    with pytest.raises(FdspError, match="both read"):
        GpuBank([var(s) * saw_hz(100.0), saw_hz(200.0) >> monitor(s, Meter.Peak(0.1))], sample_rate=SR)
    with pytest.raises(FdspError, match="inside a sequencer event"):
        GpuBank([event(saw_hz(100.0) >> monitor(s, Meter.Sample), 0.0, 0.1)], per_voice=False, mix=True, sample_rate=SR)
    with pytest.raises(FdspError, match="inside a slot"):
        GpuBank([slot(timer(s) | saw_hz(100.0))], sample_rate=SR)
    with pytest.raises(FdspError, match="both read"):
        GpuBank([var_fn(s, "|x| x * 2.0"), timer(s) | dc(0.0)], sample_rate=SR)
    bank = GpuBank([saw_hz(100.0 + i) for i in range(3)], per_voice=True, sample_rate=SR)
    bank.render_samples(100)
    with pytest.raises(FdspError, match="inside a crossfade"):
        bank.crossfade_voice(1, 1, 0.01, saw_hz(300.0) >> monitor(shared(), Meter.Sample))
    rows, _ = bank.render_samples(64)   # the refused crossfade left the bank running
    assert np.abs(rows).max() > 0.0

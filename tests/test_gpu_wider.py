"""GPU parity of the most recently added graph families (Net-as-node `Dag` programs, nonlinear biquads): same bar as
tests/test_gpu_jit.py (bit-exact vs the oracle through the C ABI), kept in a file that sorts after the parity tests."""
import numpy as np
import pytest

from test_gpu_jit import WIDER, run_case

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", sorted(WIDER))
def test_wider_graph_matches_oracle(name):
    b, g, o = run_case(WIDER[name], 40, 2000 + 61)
    assert g.shape == o.shape and np.isfinite(g).all() and np.abs(o).max() > 1e-4
    bad = int((g != o).sum())
    assert bad == 0, (name, bad, float(np.abs(g - o).max()), b.classes()[0]["signature"])


# ---------------------------------------------------------------- the sequencer as a bank of event voices (src/sequencer.rs)
def seq_five_events():   # tests/test_basic.rs:255-273 plus a fifth overlapping voice that starts mid-block
    from fundsp_b200.prelude import noise, sine_hz, mls, saw_hz, lowpass_hz
    from fundsp_b200.sequencer import Sequencer, Fade, ReplayMode
    q = Sequencer(0, 2, ReplayMode.All)
    q.push(0.1, 0.2, Fade.Smooth, 0.01, 0.0, noise() | sine_hz(220.0))
    q.push(0.3, 0.4, Fade.Smooth, 0.09, 0.08, sine_hz(110.0) | noise())
    q.push(0.25, 0.5, Fade.Power, 0.0, 0.01, mls() | noise())
    q.push(0.6, 0.7, Fade.Power, 0.02, 0.03, noise() | mls())
    q.push(0.31234, 0.45678, Fade.Smooth, 0.02, 0.05, (saw_hz(220.0) >> lowpass_hz(1000.0, 1.0)) | sine_hz(330.0))
    return q


def live_voice(f):
    from fundsp_b200.prelude import saw_hz, lowpass_hz
    return saw_hz(f) >> lowpass_hz(4.0 * f, 1.0)


def arp_voice(f):
    from fundsp_b200.prelude import saw_hz, lowpass_hz
    return saw_hz(f) >> lowpass_hz(3.0 * f, 1.5)


def _oracle_seq(seq, sr):
    from oracle import OracleUnit
    u = OracleUnit(seq.node())
    u.set_sample_rate(sr)
    return u


def _close(g, o):
    """Mix bar of DESIGN.md §4: the CTA-level sum associates differently from the sequencer's left fold over its active events."""
    tol = 1e-5 * np.maximum(np.abs(o), 1e-2 * np.abs(o).max())
    return bool(np.all(np.abs(g - o) <= tol))


def test_sequencer_bank_matches_oracle_sequencer():
    from fundsp_b200.bank import GpuBank
    from fundsp_b200.prelude import noise, sine_hz, mls, saw_hz, lowpass_hz
    from fundsp_b200.sequencer import Sequencer, Fade, ReplayMode
    from oracle import lib as olib
    olib().fo_set_denormal_emulation(0)
    sr = 44100.0

    build = seq_five_events

    n = int(0.75 * sr)
    b = GpuBank.from_sequencer(build(), per_voice=True, mix=True, sample_rate=sr)
    rows, mix = b.render_samples(n)
    want = _oracle_seq(build(), sr).process_many(n)
    assert np.abs(want).max() > 0.5 and _close(mix, want)
    # where only one event sounds, the mix IS that event: bit-exact (x + 0.0)
    solo = slice(int(0.1 * sr) + 2, int(0.2 * sr) - 2)
    assert np.array_equal(mix[:, solo], want[:, solo]) and np.array_equal(rows[0][:, solo], want[:, solo])
    assert abs(b.time() - n / sr) < 1e-9
    # ReplayMode::All: reset replays every event
    b.reset()
    rows2, mix2 = b.render_samples(n)
    assert np.array_equal(mix2, mix) and np.array_equal(rows2, rows)
    # process()-sized calls (64, 61, 7, ...) walk the same blocks as the oracle's process calls
    b.reset()
    u = _oracle_seq(build(), sr)
    sizes = [64, 61, 7, 64, 1, 33] * 60
    for k, sz in enumerate(sizes):
        got = b.process(sz)
        exp = u.process(sz)
        assert _close(got, exp), (k, sz)


def seq_loop_events(loop_samples, sr):
    """A `Sequencer::new(0, 1, ReplayMode::Loop(t))`: the event of the reference's own loop test scaled to the period (tests/test_basic.rs:730-765: it
    straddles the loop point and continues into the next period), notes that end and start again every period (their units are reset), a unit with
    delay lines, fades of both kinds, an event that starts at 0 and one that outlasts a whole period."""
    from fundsp_b200.prelude import dc, noise, sine_hz, saw_hz, moog_hz, lowpass_hz, delay, pass_
    from fundsp_b200.sequencer import Sequencer, Fade, ReplayMode
    T = loop_samples / sr
    q = Sequencer(0, 1, ReplayMode.Loop(T))
    q.push(12.0 / 79.0 * T, 89.0 / 79.0 * T, Fade.Smooth, 0.0, 0.0, dc(0.25))
    q.push(0.10 * T, 0.45 * T, Fade.Smooth, 0.05 * T, 0.10 * T, sine_hz(440.0))
    q.push(0.30 * T, 0.80 * T, Fade.Power, 0.02 * T, 0.03 * T, noise().seed(3) >> (pass_() & delay(0.0007)) >> lowpass_hz(900.0, 1.0))
    q.push(0.0, 0.20 * T, Fade.Smooth, 0.0, 0.05 * T, saw_hz(300.0) >> moog_hz(1200.0, 0.4))
    q.push(0.60 * T, 1.90 * T, Fade.Power, 0.10 * T, 0.20 * T, sine_hz(660.0) * 0.5)
    return q


@pytest.mark.parametrize("loop_samples,sr", [(79, 44100.0), (600, 44100.0), (1024, 44100.0), (3001, 44100.0), (600, 48000.0), (1024, 48000.0)])
def test_looping_sequencer_bank_matches_oracle_sequencer(loop_samples, sr):
    """ReplayMode::Loop on the device (`Event<X>` wraps its own clock, shifts a sounding event by the period, resets the unit of a finished one
    from the class's reset image): per-voice rows bit-exact against one-event oracle Sequencers of the same mode, the mix against the
    whole oracle Sequencer, over many periods in one launch and through process()-sized calls. The block path is the reference's as written
    (src/sequencer.rs:845-872: the samples of a 64-block behind the wrap are rendered into a scratch buffer and never delivered)."""
    from fundsp_b200.bank import GpuBank
    from oracle import OracleUnit, lib as olib
    olib().fo_set_denormal_emulation(0)
    # sr = 44100 is the construction-time rate. At 48 kHz the sequencer is RE-RATED after its events were pushed, which the reference turns into
    # a shift of every event by one loop period for the first pass (Sequencer::set_sample_rate :685-701 moves the ready events to `active`, then
    # reset() in loop mode moves active events back by the loop point): restated by the host lowering (graph.cpp EventN::set_sample_rate).
    n = max(64 * 40 + 37, int(3.3 * loop_samples))
    q = seq_loop_events(loop_samples, sr)
    b = GpuBank.from_sequencer(q, per_voice=True, mix=True, sample_rate=sr)
    rows, mix = b.render_samples(n)
    for v, ev in enumerate(seq_loop_events(loop_samples, sr).voices()):
        u = OracleUnit(ev); u.set_sample_rate(sr)
        want_v = u.process_many(n)
        assert np.abs(want_v).max() > 1e-3, v
        assert np.array_equal(rows[v], want_v), (loop_samples, v, int((rows[v] != want_v).sum()), float(np.abs(rows[v] - want_v).max()))
    u = _oracle_seq(seq_loop_events(loop_samples, sr), sr)
    want = u.process_many(n)
    assert _close(mix, want)
    assert abs(b.time() - olib().fo_sequencer_time(u.h)) < 1e-12, (b.time(), olib().fo_sequencer_time(u.h))
    # more than one period must actually have been played: the second period carries sound
    assert np.abs(want[:, loop_samples + 64:2 * loop_samples]).max() > 1e-3
    # process()-sized calls: blocks that wrap in the middle, at their first sample, not at all
    b2 = GpuBank.from_sequencer(seq_loop_events(loop_samples, sr), per_voice=False, mix=True, sample_rate=sr)
    u2 = _oracle_seq(seq_loop_events(loop_samples, sr), sr)
    for k, sz in enumerate([64, 61, 7, 64, 1, 33, 64, 64] * 12):
        got, exp = b2.process(sz), u2.process(sz)
        assert _close(got, exp), (loop_samples, k, sz)
    assert abs(b2.time() - olib().fo_sequencer_time(u2.h)) < 1e-12
    # edits and pushes into a running looping bank are refused, not mis-rendered
    from fundsp_b200.capi import FdspError
    with pytest.raises(FdspError):
        b.edit_event(0, 0.001, 0.0)


def test_sequencer_bank_live_edit_and_push():
    from fundsp_b200.bank import GpuBank
    from fundsp_b200.prelude import dc, sine_hz, saw_hz, lowpass_hz
    from fundsp_b200.sequencer import Sequencer, Fade, ReplayMode, event
    from oracle import OracleBackend, lib as olib
    L = olib()
    L.fo_set_denormal_emulation(0)
    sr = 44100.0
    voice = live_voice
    q = Sequencer(0, 1, ReplayMode.None_)
    e0 = q.push(0.0, 10.0, Fade.Smooth, 0.001, 0.0, voice(110.0))          # a held note, released by a later edit
    q.push(0.01, 0.02, Fade.Smooth, 0.001, 0.002, voice(220.0))             # a short note whose slot is reused
    b = GpuBank.from_sequencer(q, per_voice=False, mix=True, sample_rate=sr)
    u = _oracle_seq(q, sr)
    be = OracleBackend()
    n1 = 64 * 30                                                            # 43.5 ms in: the short note has ended
    g1 = b.render_samples(n1)[1]; o1 = u.process_many(n1)
    assert _close(g1, o1)
    # a note of a class the bank does not have yet: no slot to take over, the bank grows while the held note keeps sounding
    ta = b.time() + 0.001
    grown = b.push_event(event(sine_hz(500.0) * 0.5, ta, ta + 0.01, Fade.Power, 0.002, 0.002))
    assert grown == 2 and b.voices() == 3 and len(b.classes()) == 2
    L.fo_sequencer_push(u.h, ta, ta + 0.01, 0, 0.002, 0.002, (sine_hz(500.0) * 0.5).lower(be))
    ga = b.render_samples(64 * 4)[1]; oa = u.process_many(64 * 4)
    assert np.abs(oa).max() > 0.1 and _close(ga, oa)                       # the held note went on seamlessly, the newcomer started on time
    # release the held note: Sequencer::edit(id, end_time, fade_out) on both
    t_end = b.time() + 0.02
    b.edit_event(e0, t_end, 0.015)
    L.fo_sequencer_edit(u.h, 1, t_end, 0.015)                               # oracle event ids count from 1 in push order
    # note-on while running: the new event takes the finished note's slot and starts its clock at the bank's time
    t0 = b.time() + 0.005
    slot = b.push_event(event(voice(330.0), t0, t0 + 0.03, Fade.Smooth, 0.002, 0.004))
    assert slot == 1
    L.fo_sequencer_push(u.h, t0, t0 + 0.03, 1, 0.002, 0.004, voice(330.0).lower(be))
    n2 = 64 * 40 + 17
    g2 = b.render_samples(n2)[1]; o2 = u.process_many(n2)
    assert np.abs(o2).max() > 0.1 and _close(g2, o2)
    assert not g2[:, int((0.02 + 0.03 + 0.005) * sr):].any()                # everything has ended (times are relative to the start of g2)
    assert b.push_event(event(voice(440.0), b.time() + 1.0, b.time() + 2.0)) in (0, 1)   # both saw voices have finished: a slot is reused


def test_push_event_grows_a_bank_whose_render_is_still_running():
    """A note-on that grows the bank right behind a render_device call nobody has synchronised: the running state is read back behind that
    render. Per-voice rows bit for bit against a twin bank whose render was synchronised before the same push."""
    import ctypes
    from fundsp_b200.bank import GpuBank
    from fundsp_b200.prelude import sine_hz
    from fundsp_b200.sequencer import Sequencer, Fade, ReplayMode, event
    from test_gpu_mix import MOCK
    sr, n1, n2 = 44100.0, 64 * 30 + 5, 64 * 20 + 3

    def build():
        q = Sequencer(0, 1, ReplayMode.None_)
        q.push(0.0, 10.0, Fade.Smooth, 0.001, 0.0, live_voice(110.0))
        q.push(0.0, 10.0, Fade.Power, 0.002, 0.0, arp_voice(165.0))
        return GpuBank.from_sequencer(q, per_voice=True, mix=True, sample_rate=sr)

    a, b = build(), build()
    rows = 2 * a.voice_outputs()
    if MOCK:   # (device memory is host memory on the mock device)
        out, mix = np.full((rows, n1), np.nan, np.float32), np.full((1, n1), np.nan, np.float32)
        ptrs, fetch = (out.ctypes.data, mix.ctypes.data), lambda: (out, mix)
    else:
        import torch
        out_d = torch.full((rows, n1), float("nan"), device="cuda"); mix_d = torch.full((1, n1), float("nan"), device="cuda")
        torch.cuda.synchronize()
        ptrs, fetch = (out_d.data_ptr(), mix_d.data_ptr()), lambda: (out_d.cpu().numpy(), mix_d.cpu().numpy())
    a.render_device(n1, out_ptr=ptrs[0], out_stride=n1, mix_ptr=ptrs[1], mix_stride=n1, sync=False)
    rb, mb = b.render_samples(n1)
    t = b.time() + 0.001
    assert a.push_event(event(sine_hz(500.0) * 0.5, t, t + 0.02, Fade.Power, 0.002, 0.002)) == 2
    assert b.push_event(event(sine_hz(500.0) * 0.5, t, t + 0.02, Fade.Power, 0.002, 0.002)) == 2
    ra, ma = fetch()
    assert np.array_equal(ra, rb.reshape(ra.shape)) and np.array_equal(ma, mb)
    ra2, ma2 = a.render_samples(n2)
    rb2, mb2 = b.render_samples(n2)
    assert np.abs(rb2).max() > 0.1 and np.array_equal(ra2, rb2) and np.array_equal(ma2, mb2)


def test_gpu_sequencer_note_ons_while_running():
    """An arpeggio played live: every 1024 samples a note-on (push_relative) with a short fade, eight reserved voices that the notes
    cycle through as earlier notes finish; the oracle Sequencer receives the same calls at the same times."""
    from fundsp_b200.prelude import saw_hz, lowpass_hz
    from fundsp_b200.sequencer import GpuSequencer, Fade, ReplayMode
    from oracle import OracleBackend, OracleUnit, lib as olib
    L = olib()
    L.fo_set_denormal_emulation(0)
    sr = 44100.0
    voice = arp_voice
    g = GpuSequencer(1, ReplayMode.None_, sample_rate=sr)
    g.reserve(voice(100.0), 8)
    u = OracleUnit(L.fo_sequencer(0, 1, 1, 0.0))
    be = OracleBackend()
    got, want = [], []
    for k in range(24):
        f = 110.0 * 2.0 ** ((k * 7 % 12) / 12.0)
        dur = 0.05 + 0.01 * (k % 5)                                   # up to four notes overlap
        g.push_relative(0.003, 0.003 + dur, Fade.Smooth, 0.002, 0.01, voice(f))
        L.fo_sequencer_push_relative(u.h, 0.003, 0.003 + dur, 1, 0.002, 0.01, voice(f).lower(be))
        got.append(g.render(1024)); want.append(u.process_many(1024))
        assert abs(g.time() - L.fo_sequencer_time(u.h)) < 1e-12
    got, want = np.concatenate(got, axis=1), np.concatenate(want, axis=1)
    assert np.abs(want).max() > 0.5 and _close(got, want)
    g.reset()                                                         # ReplayMode::None: emptied
    assert not g.render(2048).any()


def test_gpu_sequencer_late_edit_of_a_finished_event_is_ignored():
    """A note-off that arrives after its note has ended — and after another note has taken over the voice — must not touch the new note
    (the reference ignores edits of past events in ReplayMode::None, src/sequencer.rs:466-476)."""
    from fundsp_b200.sequencer import GpuSequencer, Fade, ReplayMode
    from oracle import OracleBackend, OracleUnit, lib as olib
    L = olib()
    L.fo_set_denormal_emulation(0)
    sr = 44100.0
    g = GpuSequencer(1, ReplayMode.None_, sample_rate=sr)
    g.reserve(arp_voice(100.0), 1)                                    # ONE voice: the second note must reuse it
    u = OracleUnit(L.fo_sequencer(0, 1, 1, 0.0))
    be = OracleBackend()
    got, want = [g.render(64)], [u.process_many(64)]                 # the sequencer runs: from here on a push takes over a finished voice
    a = g.push_relative(0.0, 0.01, Fade.Smooth, 0.001, 0.001, arp_voice(220.0))
    ua = L.fo_sequencer_push_relative(u.h, 0.0, 0.01, 1, 0.001, 0.001, arp_voice(220.0).lower(be))
    got.append(g.render(1024)); want.append(u.process_many(1024))    # the first note (441 samples) has ended
    b = g.push_relative(0.0, 0.05, Fade.Smooth, 0.001, 0.001, arp_voice(330.0))
    L.fo_sequencer_push_relative(u.h, 0.0, 0.05, 1, 0.001, 0.001, arp_voice(330.0).lower(be))
    assert g.voice_of[b] == 0 and a not in g.voice_of                 # the finished note's id no longer maps to the voice
    g.edit_relative(a, 0.0, 0.0)                                      # late note-off of the first note
    L.fo_sequencer_edit_relative(u.h, ua, 0.0, 0.0)
    got.append(g.render(4096)); want.append(u.process_many(4096))
    got, want = np.concatenate(got, axis=1), np.concatenate(want, axis=1)
    assert np.abs(want[:, 1088:3000]).max() > 0.1 and _close(got, want)    # the second note sounds in full
    g.edit(12345, 0.0, 0.0)                                           # an id that never existed: no-op


def test_slot_crossfades_to_a_new_unit():
    """Slot / SlotBackend (src/slot.rs) as voices: units replaced with a crossfade while the bank runs, no new program built. Per-voice rows
    are bit-exact against oracle Slots that receive the same `set` calls at the same times."""
    from fundsp_b200.bank import GpuBank
    from fundsp_b200.capi import FdspError
    from fundsp_b200.prelude import saw_hz, lowpass_hz, sine_hz
    from fundsp_b200.sequencer import slot, Fade
    from oracle import OracleBackend, OracleUnit, lib as olib
    L = olib()
    L.fo_set_denormal_emulation(0)
    sr = 44100.0                                   # (the reference does not re-rate a unit that arrives through Slot::set)
    voice = lambda f, q=1.0: saw_hz(f) >> lowpass_hz(3.0 * f, q)
    V = 6
    b = GpuBank([slot(voice(110.0 * (k + 1))) for k in range(V)], per_voice=True, mix=False, sample_rate=sr)
    us = [OracleUnit(slot(voice(110.0 * (k + 1)))) for k in range(V)]
    be = OracleBackend()

    def both(n):
        g = b.render_samples(n)[0]
        o = np.stack([u.process_many(n) for u in us])
        assert np.array_equal(g, o), (int((g != o).sum()), float(np.abs(g - o).max()))
        return g

    both(64 * 5)
    b.slot_set(2, Fade.Smooth, 0.01, voice(500.0, 2.0)); L.fo_slot_set(us[2].h, 1, 0.01, voice(500.0, 2.0).lower(be))
    b.slot_set(4, Fade.Power, 0.003, voice(77.0)); L.fo_slot_set(us[4].h, 0, 0.003, voice(77.0).lower(be))
    g = both(64 * 3 + 17)                          # mid-fade, ragged block
    # a set while the voice is still fading is parked as `latest` (src/slot.rs:142-150), a newer one replaces it, and the voice starts fading to it
    # in the block after its running fade has ended: the bank cuts the launch there (the fade of voice 2 ends inside the next render)
    b.slot_set(2, Fade.Smooth, 0.01, voice(300.0)); L.fo_slot_set(us[2].h, 1, 0.01, voice(300.0).lower(be))
    b.slot_set(2, Fade.Power, 0.004, voice(333.0, 3.0)); L.fo_slot_set(us[2].h, 0, 0.004, voice(333.0, 3.0).lower(be))   # replaces the parked one
    with pytest.raises(FdspError):
        b.slot_set(1, Fade.Smooth, 0.01, sine_hz(300.0))   # another graph class
    with pytest.raises(FdspError):
        b.slot_set(2, Fade.Smooth, 0.01, sine_hz(300.0))   # ... also refused at once when it would only be parked
    both(64 * 9)                                   # first fades end; voice 2 goes on to its parked unit
    both(64 * 2 + 9); both(31); both(64 * 6)       # (ragged calls across the second fade)
    b.slot_set(2, Fade.Power, 0.002, voice(250.0)); L.fo_slot_set(us[2].h, 0, 0.002, voice(250.0).lower(be))   # the roles have swapped: the other instance takes it
    both(64 * 4 + 5)
    # reset with an update parked behind a running fade adopts the parked (latest) unit (:156-172)
    b.slot_set(3, Fade.Smooth, 0.02, voice(90.0)); L.fo_slot_set(us[3].h, 1, 0.02, voice(90.0).lower(be))
    both(64 * 2)
    b.slot_set(3, Fade.Smooth, 0.02, voice(700.0, 4.0)); L.fo_slot_set(us[3].h, 1, 0.02, voice(700.0, 4.0).lower(be))   # parked
    both(64)
    b.reset()                                      # reset adopts the newest units
    for u in us:
        u.reset()
    assert np.abs(both(64 * 3)).max() > 0.1
    # process()-sized calls with an update parked: armed between two calls
    b.slot_set(0, Fade.Power, 0.003, voice(123.0)); L.fo_slot_set(us[0].h, 0, 0.003, voice(123.0).lower(be))
    both(64)
    b.slot_set(0, Fade.Smooth, 0.002, voice(456.0)); L.fo_slot_set(us[0].h, 1, 0.002, voice(456.0).lower(be))   # parked
    for size in (64, 64, 61, 64, 7, 64, 64, 64):
        both(size)


def test_bank_grows_with_a_new_waveform_and_keeps_running_state():
    """fdsp_bank_add_voice: voices with delay lines and filter state keep running bit for bit while the bank is rebuilt around them, and
    a newcomer may bring a wavetable the bank had not loaded."""
    from fundsp_b200.bank import GpuBank
    from fundsp_b200.prelude import sine_hz, noise, feedback, delay, lowpass_hz, square_hz, organ_hz
    from oracle import OracleUnit, lib as olib
    olib().fo_set_denormal_emulation(0)
    sr = 48000.0
    echo = lambda i: noise().seed(i) * 0.3 >> lowpass_hz(900.0 + 100.0 * i, 1.0) >> feedback(delay(0.002 + 0.0005 * i) * 0.6)
    voices = [sine_hz(200.0 + 10.0 * i) for i in range(3)] + [echo(i) for i in range(3)]
    b = GpuBank(voices, per_voice=True, mix=False, sample_rate=sr)
    us = [OracleUnit(v) for v in voices]
    for u in us:
        u.set_sample_rate(sr)

    def both(n):
        g = b.render_samples(n)[0]
        o = np.stack([u.process_many(n) for u in us])
        assert np.array_equal(g, o), (int((g != o).sum()), float(np.abs(g - o).max()))

    both(64 * 7 + 3)
    for newcomer in (square_hz(330.0) >> lowpass_hz(2000.0, 1.0), echo(7), organ_hz(150.0)):   # a new class with a table, an existing class, another table
        v = b.add_voice(newcomer)
        assert v == len(us) and b.voices() == len(us) + 1
        u = OracleUnit(newcomer); u.set_sample_rate(sr); us.append(u)
        both(64 * 5 + 11)
    assert len(b.classes()) == 7                  # sine, four echo delay lengths (class-uniform words), square+filter, organ
    b.reset()
    for u in us:
        u.reset()
    both(64 * 4)


def test_event_workload_of_the_bench_matches_oracle():
    """`bench.py --workload saw_svf_events`: the headline voices as held sequencer events (start within 0.5 s, fade-in 5 ms)."""
    from fundsp_b200 import workloads
    from fundsp_b200.bank import GpuBank
    from oracle import lib as olib, oracle_bank_render
    olib().fo_set_denormal_emulation(0)
    V, n, sr = 64, 28800, 48000.0
    b = GpuBank(workloads.build("saw_svf_events", V), per_voice=True, mix=True, sample_rate=sr)
    rows, mix = b.render_samples(n)
    ref, _ = oracle_bank_render(workloads.build("saw_svf_events", V), sr, n, threads=4)
    assert np.array_equal(rows, ref) and np.abs(ref[:, :, -64:]).max(axis=(1, 2)).min() > 0.0     # every note has started and is held
    assert _close(mix, ref.astype(np.float64).sum(0).astype(np.float32))
    rows2, _ = b.render_samples(4800)                 # steady state: every block is a whole block of every event (X's own group form)
    cont = oracle_bank_render(workloads.build("saw_svf_events", V), sr, n + 4800, threads=4)[0][:, :, n:]
    assert np.array_equal(rows2, cont)


def test_gpu_sequencer_replay_all_keeps_every_event():
    """ReplayMode::All: events pushed while running are added (never written over a finished one), so a reset replays all of them."""
    from fundsp_b200.sequencer import GpuSequencer, Fade, ReplayMode
    from oracle import OracleBackend, OracleUnit, lib as olib
    L = olib()
    L.fo_set_denormal_emulation(0)
    sr = 44100.0
    g = GpuSequencer(1, ReplayMode.All, sample_rate=sr)
    u = OracleUnit(L.fo_sequencer(0, 1, 0, 0.0))
    be = OracleBackend()
    def push(start, end, f):
        g.push(start, end, Fade.Smooth, 0.002, 0.004, arp_voice(f))
        L.fo_sequencer_push(u.h, start, end, 1, 0.002, 0.004, arp_voice(f).lower(be))
    push(0.0, 0.02, 220.0)
    a = g.render(64 * 20); b = u.process_many(64 * 20)             # the first note has ended
    assert _close(a, b) and np.abs(b).max() > 0.1
    push(g.time() + 0.001, g.time() + 0.02, 330.0)                  # a second note, pushed into the running sequencer
    a = g.render(64 * 20); b = u.process_many(64 * 20)
    assert _close(a, b) and np.abs(b).max() > 0.1 and g.bank.voices() == 2
    g.reset(); u.reset()                                            # both notes replay
    a = g.render(64 * 45); b = u.process_many(64 * 45)
    assert _close(a, b) and np.abs(b[:, :64 * 20]).max() > 0.1 and np.abs(b[:, 64 * 21:]).max() > 0.1


def test_net_bank_replace_and_remove_vertices_across_classes():
    """Net::replace / Net::remove (src/net.rs:351-404,460-470) on a RUNNING bank made from a Net: a vertex gets a unit of ANOTHER graph class
    (the voice moves to that class — compiled on the spot if new — while every other voice keeps its running state and the mix keeps the Net's
    association order), another vertex is removed (its connections carry zeros). Rows against an unedited twin bank and fresh oracle units."""
    from fundsp_b200 import workloads
    from fundsp_b200.bank import GpuBank
    from fundsp_b200.net import voice_net
    from fundsp_b200.prelude import moog_hz, pan, noise, lowpass_hz
    from oracle import OracleUnit, lib as olib
    olib().fo_set_denormal_emulation(0)
    SR = 48000.0
    V, n1, n2 = 21, 1000 + 7, 1500
    mk = lambda: voice_net([workloads.net_voice(i) for i in range(V)])
    b = GpuBank.from_net(mk(), per_voice=True, mix=True, sample_rate=SR)
    twin = GpuBank.from_net(mk(), per_voice=True, mix=True, sample_rate=SR)
    b.render_samples(n1); twin.render_samples(n1)
    newcomer = lambda: noise().seed(77) >> lowpass_hz(700.0, 2.0) >> moog_hz(900.0, 0.3) >> pan(0.25)     # a class the bank does not have yet
    b.replace_voice(4, newcomer())
    b.replace_voice(9, workloads.net_voice(2))                                  # an existing class (voice 9 was class B)
    b.remove_voice(13)           # (fdsp_bank_voice_of_vertex maps a NodeId to the voice index, see test_net_bank_setting_by_node_id)
    assert len(b.classes()) >= 5
    rows, mix = b.render_samples(n2)
    want, _ = twin.render_samples(n2)
    changed = [v for v in range(V) if not np.array_equal(rows[v], want[v])]
    assert changed == [4, 9, 13], changed                                   # every other voice just continues
    assert not rows[13].any()
    for v, g in ((4, newcomer()), (9, workloads.net_voice(2))):
        u = OracleUnit(g); u.set_sample_rate(float(np.float32(SR)))          # (a Net hands its units the f32-rounded rate)
        assert np.array_equal(rows[v], u.process_many(n2)), v
    ref = rows.astype(np.float64).sum(axis=0)
    assert np.abs(mix - ref).max() <= 1e-5 * max(1.0, np.abs(rows).sum(axis=0).max())
    b.reset()                                                               # reset keeps the edited net
    r2, _ = b.render_samples(200)
    u = OracleUnit(newcomer()); u.set_sample_rate(float(np.float32(SR)))
    assert not r2[13].any() and np.array_equal(r2[4], u.process_many(200))


def test_net_bank_crossfades_vertices_across_classes():
    """Net::crossfade (src/net.rs:480-504, src/vertex.rs:138-229) on a RUNNING bank made from a Net: a vertex fades to a unit of ANOTHER graph class
    (device: Xfade<X, Y>; the old unit keeps running inside the new class with its state and delay lines carried over), with both curves, fades
    that end inside a block, process()-sized calls during the fade, a second crossfade of a vertex that has arrived, and crossfades parked behind a
    running one (`latest`). The mix equals the oracle Net that receives the same `crossfade` calls bit for bit (it is summed in the Net's own order)."""
    from fundsp_b200 import workloads
    from fundsp_b200.bank import GpuBank
    from fundsp_b200.capi import FdspError
    from fundsp_b200.net import voice_net
    from fundsp_b200.prelude import moog_hz, pan, noise, lowpass_hz, saw_hz, delay, pass_
    from fundsp_b200.sequencer import Fade
    from oracle import OracleBackend, OracleUnit, lib as olib
    L = olib(); L.fo_set_denormal_emulation(0)
    SR = 48000.0
    V = 13
    mk = lambda: voice_net([workloads.net_voice(i) for i in range(V)])
    b = GpuBank.from_net(mk(), per_voice=True, mix=True, sample_rate=SR)
    twin = GpuBank.from_net(mk(), per_voice=True, mix=True, sample_rate=SR)
    u = OracleUnit(mk().node()); u.set_sample_rate(SR)
    be = OracleBackend()
    vertex_of = {b.voice_of_vertex(x): x for x in range(mk().size()) if b.voice_of_vertex(x) >= 0}
    assert sorted(vertex_of) == list(range(V))

    def both(n):
        rows, mix = b.render_samples(n)
        want = u.process_many(n)
        assert np.array_equal(mix, want), (n, int((mix != want).sum()), float(np.abs(mix - want).max()))
        return rows

    both(1000 + 7); twin.render_samples(1000 + 7)
    new_a = lambda: noise().seed(77) >> (pass_() & delay(0.0004)) >> lowpass_hz(700.0, 2.0) >> moog_hz(900.0, 0.3) >> pan(0.25)   # a class the bank does not have
    new_c = lambda: workloads.net_voice(2 + 4 * 5)                                                                                  # a class it has (noise >> bandpass >> pan)
    b.crossfade_voice(4, Fade.Smooth, 0.01, new_a());   L.fo_net_crossfade(u.h, vertex_of[4], Fade.Smooth, 0.01, new_a().lower(be))
    b.crossfade_voice(9, Fade.Power, 0.0333, new_c());  L.fo_net_crossfade(u.h, vertex_of[9], Fade.Power, 0.0333, new_c().lower(be))
    assert any("Xfade<" in c["signature"] for c in b.classes())
    rows = both(300)                                                      # inside both fades
    want_rows, _ = twin.render_samples(300)
    changed = [v for v in range(V) if not np.array_equal(rows[v], want_rows[v])]
    assert changed == [4, 9], changed                                    # every other voice just continues
    # a crossfade of a vertex that is still fading waits as `latest` (src/vertex.rs:203-218; a newer one replaces it) and starts in the block after
    # the running fade has ended: the bank finds that block, cuts its launch there and moves the voice to the class Xfade<new_a, new_c>
    b.crossfade_voice(4, Fade.Power, 0.5, workloads.net_voice(3)); L.fo_net_crossfade(u.h, vertex_of[4], Fade.Power, 0.5, workloads.net_voice(3).lower(be))
    b.crossfade_voice(4, Fade.Smooth, 0.01, new_c()); L.fo_net_crossfade(u.h, vertex_of[4], Fade.Smooth, 0.01, new_c().lower(be))   # replaces the parked one
    for sz in (64, 61, 7, 64, 64, 33, 64):                                # the 480-sample fade of voice 4 ends inside one of these blocks
        got, exp = b.process(sz), u.process(sz)
        assert np.array_equal(got, exp), sz
    both(64 * 30 + 5)                                                     # past the end of the second fade (1598 samples)
    # a vertex that has arrived fades again, from the unit it arrived at
    b.crossfade_voice(4, Fade.Power, 0.004, workloads.net_voice(1)); L.fo_net_crossfade(u.h, vertex_of[4], Fade.Power, 0.004, workloads.net_voice(1).lower(be))
    both(500)
    # a parked crossfade whose turn comes in the MIDDLE of a long render: the launch is cut behind the block in which the running fade ends
    b.crossfade_voice(9, Fade.Smooth, 0.005, workloads.net_voice(0)); L.fo_net_crossfade(u.h, vertex_of[9], Fade.Smooth, 0.005, workloads.net_voice(0).lower(be))
    both(64)
    b.crossfade_voice(9, Fade.Power, 0.003, new_a()); L.fo_net_crossfade(u.h, vertex_of[9], Fade.Power, 0.003, new_a().lower(be))   # parked: 176 samples of the first fade are left
    both(64 * 20 + 3)
    # reset: the edited net, every vertex at its newest unit
    b.reset(); u.reset()
    r2 = both(300)
    assert np.abs(r2[4]).max() > 1e-3


# ---------------------------------------------------------------- AudioUnit::reset where the reference's reset is NOT "back to the constructed state"
@pytest.mark.parametrize("name", ["reverb3_lowpass_loop", "limiters"])
def test_bank_reset_leaves_alone_what_the_reference_reset_leaves_alone(name):
    """Reverb::reset (src/reverb.rs:215-228) resets its eight loop blocks and the feedback sample but NOT its four pre-delay allpasses;
    Limiter::reset (src/dynamics.rs:181-195) is set_sample_rate: index, reducer and buffer are cleared, the follower keeps its state.
    `fdsp_bank_reset` follows both (Lowering::keepS / keepD): render, reset, render equals the oracle units doing the same, bit for bit — and
    the second render differs from the first (something did survive the reset) for the reverb."""
    from fundsp_b200.bank import GpuBank
    from oracle import OracleUnit, lib as olib
    from test_gpu_jit import CASES, SR
    mk = {**CASES, **WIDER}[name]
    olib().fo_set_denormal_emulation(0)
    V, n1, n2 = 12, 1500 + 37, 900
    b = GpuBank([mk(i) for i in range(V)], per_voice=True, sample_rate=SR)
    g1, _ = b.render_samples(n1)
    b.reset()
    g2, _ = b.render_samples(n2)
    for v in (0, 5, V - 1):
        u = OracleUnit(mk(v)); u.set_sample_rate(SR)
        o1 = u.process_many(n1)
        u.reset()
        o2 = u.process_many(n2)
        assert np.array_equal(g1[v], o1), (name, v, "before the reset")
        assert np.array_equal(g2[v], o2), (name, v, "after the reset", int((g2[v] != o2).sum()))
    if name.startswith("reverb3"):
        assert not np.array_equal(g2, g1[..., :n2])   # the pre-delay allpasses were still ringing

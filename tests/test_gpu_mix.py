"""The mix-down of every bank path, bit for bit against a float32 model of its summation order, and against the f64 sum of the rows.

Every mix path is deterministic: the order of its additions is fixed by the code. `mix_model` writes that order down in numpy float32
(IEEE single, one rounding per addition), so a mix is compared with `np.array_equal` and a dropped, doubled or misplaced voice, a stale
tile row or a missed accumulate is caught whatever its size. The order (DESIGN.md §2, §4):

- classes in order of first appearance, voices in bank order inside a class;
- CTA shape: `bank_grid(V, 128, SMs)` (csrc/dsp/bank_args.h), or `staged_grid` for a stage-pipelined class (csrc/host/bank.cpp
  `use_staged`: stages >= 2, launch length >= 256, V <= 32 SMs; 32 voices per CTA, 128 with FDSP_STAGED_W=128; the kernel is 32 wide
  whenever vpc <= 32);
- CTA partial (`cta_partials`): column j of CTA b holds voice b * vpc + j, or +0.0; HALF = NT / 2, QN = HALF / 4; thread h of a row has
  four accumulators, accumulator q starts at column h * HALF + ((q + h) * QN mod HALF) and left-folds QN columns;
  s_h = (a0 + a1) + (a2 + a3), partial = s_0 + s_1;
- class fold: the partials left-folded in CTA order from partial 0 (mix_reduce_kernel, the fused finish of short launches, the resident
  kernel); a two-stage (FDN) class has one partial per voice, so its fold is the left fold of its voices;
- bank: the first class writes the mix, every later class adds its fold, in class order. A pipelined bank (a two-stage class with a dry
  program) starts from a zeroed mix, adds the fold of every other class in class order, then those of its two-stage classes, one chunk
  late, in class order.

The mix bits depend on the SM count through `bank_grid`: the model takes it from the device (132 on the CPU mock device).
Every case also meets the f64 bound d * u * sum_v |x_v(t)| (u = 2^-24, d = the longest addition chain of the model)."""
import functools
import os
import re

import numpy as np
import pytest

from fundsp_b200 import capi, workloads
from fundsp_b200.prelude import *  # noqa: F401,F403
from oracle import lib as olib, oracle_bank_render

pytestmark = pytest.mark.gpu
SR = 48000.0
MOCK = "mock" in os.environ.get("FDSP_B200_LIB", "")
MOCK_BUDGET = 6_000_000          # voice-channel-samples of one case on the CPU mock device (it walks every voice serially)
U = 2.0 ** -24
TIME_CHUNK, PIPE_CHUNK = 16384, 2048
REV = "Pipe<Pipe<MultiSplit<2,16>,Feedback<1,Multi<30,0,32,Pipe<Delay,Fir<3>>>>>,Binop<2,Multi<31,0,32,Panner<1>>,Constant<2>>>"


@functools.lru_cache(None)
def sms():
    """SMs of device 0: what bank_grid sizes the CTA shapes by."""
    if MOCK:
        return 132                # tests/cpp/mock/cuda_runtime.h
    # the driver API, not torch: importing torch first would put its own libnvrtc in the process, and the JIT cache keys its entries
    # by the NVRTC version
    import ctypes as C
    cu = C.CDLL("libcuda.so.1")
    dev, n = C.c_int(), C.c_int()
    assert cu.cuInit(0) == 0 and cu.cuDeviceGet(C.byref(dev), 0) == 0
    assert cu.cuDeviceGetAttribute(C.byref(n), 16, dev) == 0   # CU_DEVICE_ATTRIBUTE_MULTIPROCESSOR_COUNT
    return n.value


def vcount(label):
    """Voice counts are written in SMs: "32s+1" is 32 voices per SM plus one."""
    m = re.fullmatch(r"(\d+)(?:s([+-]\d+)?)?", label)
    return int(m.group(1)) * sms() + int(m.group(2) or 0) if "s" in label else int(label)


# ---------------------------------------------------------------- the model
def bank_grid(V, nt, sms):
    grid = (V + nt - 1) // nt
    if V >= sms * 32:
        grid = (grid + sms - 1) // sms * sms
    grid = max(grid, 1)
    vpc = (V + grid - 1) // grid
    return (V + vpc - 1) // vpc, vpc


def staged_grid(V, sms, w128):
    if V <= sms * 32 and not w128:
        return (V + 31) // 32, 32
    return bank_grid(V, 128, sms)


def cta_partials(x, vpc, grid, nt):
    """[V, C, n] rows of one class -> [grid, C, n] CTA partials in the association of the mix tile."""
    V = x.shape[0]
    half = nt // 2
    qn = max(1, half // 4)
    zero = np.zeros((grid,) + x.shape[1:], np.float32)
    b = np.arange(grid)

    def col(j):
        if j >= vpc:
            return zero
        v = b * vpc + j
        ok = v < V
        out = zero.copy()
        out[ok] = x[v[ok]]
        return out

    s = []
    for h in (0, 1):
        acc = []
        for q in range(4):
            c0 = h * half + (q * qn + h * qn) % half
            a = col(c0)
            for j in range(1, qn):
                a = a + col(c0 + j)
            acc.append(a)
        s.append((acc[0] + acc[1]) + (acc[2] + acc[3]))
    return s[0] + s[1]


def left_fold(p):
    s = p[0].copy()
    for i in range(1, p.shape[0]):
        s = s + p[i]
    return s


class Klass:
    def __init__(self, sig, voices, stages, nin):
        self.sig, self.voices, self.stages = sig, np.asarray(voices), stages
        wet_tail, pipe_tail = ",Bus<MultiPass<2>,Unop<3," + REV + ">>>", "," + REV + ">"
        if nin == 2 and sig in (REV, "Bus<MultiPass<2>,Unop<3," + REV + ">>"):
            self.kind = "fdn"          # reverb on the bank input: FDN kernel alone, reduced in class order
        elif sig.startswith("Pipe<") and (sig.endswith(wet_tail) or sig.endswith(pipe_tail)):
            self.kind = "fdn_dry"      # dry program -> FDN kernel: pipelined
        else:
            self.kind = "plain"


def bank_classes(bank, voices):
    """The bank's classes with their voices: grouped by signature in order of first appearance (csrc/host/bank.cpp lower_and_upload),
    checked against what the bank reports."""
    sigs = [capi.NodeHandle(v).signature() for v in voices]
    order, groups = [], {}
    for i, s in enumerate(sigs):
        if s not in groups:
            groups[s] = []
            order.append(s)
        groups[s].append(i)
    info = bank.classes()
    assert [(c["signature"], c["voices"]) for c in info] == [(s, len(groups[s])) for s in order], "class grouping differs from the bank's"
    return [Klass(s, groups[s], c["stages"], bank.inputs()) for s, c in zip(order, info)]


def is_pipelined(classes, env=os.environ):
    return "FDSP_NO_PIPELINE" not in env and any(c.kind == "fdn_dry" for c in classes)


def launch_segments(n, classes, V, C, per_voice_rows, pipelined):
    """(t0, len) of every launch of render_samples(n) (bank.cpp render_host -> render_device chunking)."""
    chunk = TIME_CHUNK
    if per_voice_rows:
        cap = (512 << 20) // (V * C * 4)
        chunk = max(64, min(TIME_CHUNK, cap // 64 * 64))
    chunk = min(chunk, (n + 63) // 64 * 64)
    ch = PIPE_CHUNK if pipelined else TIME_CHUNK
    segs = []
    for t0 in range(0, n, chunk):
        ln = min(chunk, n - t0)
        segs += [(t0 + u, min(ch, ln - u)) for u in range(0, ln, ch)]
    return segs


def class_shape(c, ln):
    """(grid, vpc, NT) of a plain class in a launch of `ln` samples."""
    V = len(c.voices)
    staged = os.environ.get("FDSP_STAGED", "1") != "0" and c.stages >= 2 and ln >= 256 and V <= sms() * 32
    if staged:
        grid, vpc = staged_grid(V, sms(), os.environ.get("FDSP_STAGED_W") == "128")
        return grid, vpc, (32 if vpc <= 32 else 128)
    grid, vpc = bank_grid(V, 128, sms())
    return grid, vpc, 128


def class_fold(x, c, ln):
    xc = x if len(c.voices) == x.shape[0] else x[c.voices]
    if c.kind != "plain":
        return left_fold(xc)
    grid, vpc, nt = class_shape(c, ln)
    return left_fold(cta_partials(xc, vpc, grid, nt))


def mix_model(rows, classes, segments, pipelined):
    """rows [V, C, n] float32 -> the mix [C, n] the bank computes, bit for bit."""
    rows = np.asarray(rows, np.float32)
    out = np.zeros(rows.shape[1:], np.float32)
    for t0, ln in segments:
        x = rows[:, :, t0:t0 + ln]
        folds = [class_fold(x, c, ln) for c in classes]
        if pipelined:
            m = np.zeros(x.shape[1:], np.float32)
            for f, c in zip(folds, classes):
                if c.kind != "fdn_dry":
                    m = m + f
            for f, c in zip(folds, classes):
                if c.kind == "fdn_dry":
                    m = m + f
        else:
            m = folds[0]
            for f in folds[1:]:
                m = m + f
        out[:, t0:t0 + ln] = m
    return out


def chain_length(classes, segments, pipelined):
    """Longest addition chain of the model: QN + 2 + grid - 1 per plain class (V - 1 for a two-stage one), + classes - 1, + 1 for a zeroed start."""
    d = 0
    for _, ln in segments:
        for c in classes:
            if c.kind == "plain":
                grid, _, nt = class_shape(c, ln)
                d = max(d, max(1, nt // 8) + 2 + grid - 1)
            else:
                d = max(d, len(c.voices) - 1)
    return d + len(classes) - 1 + (1 if pipelined else 0)


def f64_sums(rows):
    """(sum_v x_v, sum_v |x_v|) in f64, a block of voices at a time."""
    s = np.zeros(rows.shape[1:], np.float64)
    a = np.zeros(rows.shape[1:], np.float64)
    for v0 in range(0, rows.shape[0], 2048):
        blk = rows[v0:v0 + 2048].astype(np.float64)
        s += blk.sum(axis=0)
        a += np.abs(blk).sum(axis=0)
    return s, a


def check_mix(mix, rows, classes, segments, pipelined, what=""):
    expect = mix_model(rows, classes, segments, pipelined)
    assert mix.shape == expect.shape
    bad = np.argwhere(mix != expect)
    assert bad.size == 0, (what, len(bad), bad[:4].tolist(), float(np.abs(mix - expect).max()))
    s, a = f64_sums(rows)
    d = chain_length(classes, segments, pipelined)
    g = d * U / (1.0 - d * U)
    assert np.all(np.abs(expect.astype(np.float64) - s) <= g * a), (what, d, float((np.abs(expect - s) / np.maximum(a, 1e-300)).max()))
    return expect


def too_big_for_mock(V, C, n):
    return MOCK and V * C * n > MOCK_BUDGET


def Bank(voices, per_voice, mix):
    from fundsp_b200.bank import GpuBank
    return GpuBank(voices, per_voice=per_voice, mix=mix, sample_rate=SR)


def render_and_check(voices, n, inp=None, mix_only_too=True, oracle=False, voices_again=None, what=""):
    """Rows + mix of one render against the model (and the model of the oracle's rows); the mix-only bank gives the same bits."""
    b = Bank(voices, True, True)
    rows, mix = b.render_samples(n, inp)
    classes = bank_classes(b, voices)
    V, C = rows.shape[0], rows.shape[1]
    pipe = is_pipelined(classes)
    segs = launch_segments(n, classes, V, C, True, pipe)
    assert np.abs(rows).max() > 1e-3, "degenerate test signal"
    expect = check_mix(mix, rows, classes, segs, pipe, what)
    del b
    if oracle:
        olib().fo_set_denormal_emulation(0)
        o, _ = oracle_bank_render(voices_again(), SR, n, inp, threads=4)
        assert np.array_equal(mix_model(o, classes, segs, pipe), mix), (what, "model of the oracle's rows")
    if mix_only_too:
        m = Bank(voices_again() if voices_again else voices, False, True)
        _, mix2 = m.render_samples(n, inp)
        assert np.array_equal(mix2, mix), (what, "mix-only bank")
        del m
    return rows, mix, classes, segs, expect


# ---------------------------------------------------------------- channels x CTA shape
def stack_voice(k):
    """k outputs: k independent noise >> lowpass chains."""
    return lambda i: stacki(k, lambda c: white().seed(k * i + c) >> lowpass_hz(workloads.xerp(100.0, 12000.0, workloads.u(k * i + c, 0)),
                                                                               workloads.lerp(0.5, 10.0, workloads.u(k * i + c, 1))))


VOICE_OF = {1: workloads.noise_svf_voice, 2: stack_voice(2), 3: stack_voice(3), 4: stack_voice(4), 5: stack_voice(5),
            8: workloads.biquad_bank_unit}
V_ALL = ["1", "31", "33", "128", "129", "32s-1", "32s", "32s+1", "128s", "128s+1"]
V_WIDE = ["1", "33", "129", "32s-1", "32s+1", "128s+1"]
SHAPES = [(1, V, n) for V in V_ALL for n in (64 * 5 + 61,)] + [(1, V, TIME_CHUNK + 64 * 2 + 29) for V in ("33", "32s+1")] + \
         [(k, V, 64 * 5 + 61) for k in (2, 3, 4, 5, 8) for V in V_WIDE] + [(k, "129", TIME_CHUNK + 64 + 13) for k in (2, 5)]
EXACT_ORACLE = {1, 8}   # noise_svf and biquad_bank rows equal the oracle's bit for bit


@pytest.mark.parametrize("k,V,n", SHAPES)
def test_mix_tile_shapes(k, V, n):
    """Tile depths 64, 32, 16, 16, 8, 8 (1..8 outputs) over the voice counts where bank_grid changes shape."""
    V = vcount(V)
    if too_big_for_mock(V, k, n):
        pytest.skip("large for the CPU mock device")
    fn = VOICE_OF[k]
    mk = lambda: [fn(i) for i in range(V)]   # noqa: E731
    oracle = k in EXACT_ORACLE and V * k * n <= 8_000_000
    render_and_check(mk(), n, oracle=oracle, voices_again=mk, what=(k, V, n))


def _drop_check(rows, mix, classes, segs, pipe):
    """Leaving one sounding voice out of the model's input must change the expected mix; says whether the sqrt(V) bar would have caught it."""
    e = np.abs(rows).max(axis=(1, 2))
    v = int(np.argmax(e))
    r2 = rows.copy()
    r2[v] = 0.0
    perturbed = mix_model(r2, classes, segs, pipe)
    assert not np.array_equal(perturbed, mix), "one voice less must change the mix"
    V = rows.shape[0]
    s, a = f64_sums(rows)
    old_bar = 4.0 * np.sqrt(V) * U * a.max() + 1e-7
    err = float(np.abs(perturbed - s).max())
    print(f"\n[drop one voice] V={V}: |perturbed - f64| = {err:.3g}, sqrt(V) bar = {old_bar:.3g}: "
          f"{'ACCEPTED by the old bar' if err <= old_bar else 'caught by the old bar'}")


def test_big_mono_bank_one_voice_removed():
    V, n = vcount("128s+1"), 64 * 3 + 61
    if too_big_for_mock(V, 1, n):
        pytest.skip("large for the CPU mock device")
    rows, mix, classes, segs, _ = render_and_check(workloads.build("noise_svf", V), n, mix_only_too=False)
    assert V >= 16384
    _drop_check(rows, mix, classes, segs, False)


def test_65536_voice_stereo_bank_with_rows():
    """Per-voice staging of 65 536 stereo voices splits render_host into 1 024-sample chunks."""
    V, n = 65536, 1024 + 64 * 2 + 61
    if MOCK:
        pytest.skip("large for the CPU mock device")
    fn = VOICE_OF[2]
    rows, mix, classes, segs, _ = render_and_check([fn(i) for i in range(V)], n, voices_again=lambda: [fn(i) for i in range(V)])
    assert segs[0] == (0, 1024) and len(segs) == 2
    _drop_check(rows, mix, classes, segs, False)


# ---------------------------------------------------------------- short launches: fused finish into the mapped host buffer
def multi_voice(kinds):
    fns = [workloads.noise_svf_voice, workloads.saw_svf_voice, workloads.fm_voice]
    return lambda i: fns[kinds[i]](i)


def class_pattern(ncls, V, seed=5):
    rng = np.random.default_rng(seed)
    k = rng.integers(0, ncls, V)
    k[:ncls] = np.arange(ncls)[::-1]      # classes appear in the order 2, 1, 0: first appearance, not kind order
    return [int(x) for x in k]


@pytest.mark.parametrize("ncls", [1, 2, 3])
def test_short_launches_fused_finish(ncls):
    """render_samples(n <= 64) and process(size) in mix mode: the last CTA folds the partials into the mix (process: the mapped host
    buffer), and later classes accumulate. Rows from a per-voice twin bank driven with the same calls."""
    V = 300
    mk = multi_voice(class_pattern(ncls, V))
    voices = lambda: [mk(i) for i in range(V)]   # noqa: E731
    m, t = Bank(voices(), False, True), Bank(voices(), True, False)
    classes = bank_classes(m, voices())
    calls = [("r", 1), ("r", 17), ("r", 64), ("p", 64), ("p", 61), ("p", 8), ("p", 7), ("p", 1), ("r", 33), ("p", 64), ("p", 17)]
    for kind, n in calls:
        if kind == "r":
            _, mix = m.render_samples(n)
            rows, _ = t.render_samples(n)
        else:
            mix = m.process(n)
            rows = t.process(n).reshape(V, 1, n)
        check_mix(mix, rows, classes, [(0, n)], False, (ncls, kind, n))
    assert np.abs(mix).max() > 1e-3


# ---------------------------------------------------------------- the resident process() kernel
RT_CASES = {
    "in2_stereo": (lambda i: stacki(2, lambda c: pass_() * white().seed(2 * i + c) >> lowpass_hz(300.0 + 37.0 * i + 500.0 * c, 1.0 + 0.1 * c)), 200),
    "five_out": (stack_voice(5), 300),
    "mono_32s": (workloads.noise_svf_voice, "32s"),
    "mono_128s": (workloads.noise_svf_voice, "128s"),
}


@pytest.mark.parametrize("case", sorted(RT_CASES))
@pytest.mark.parametrize("rt", ["1", "0"])
def test_resident_process_kernel(case, rt, monkeypatch):
    """Shared-input staging (s_in), several tile passes per block (5 outputs: depth 8), the largest resident grid (SMs x 128 voices):
    the resident kernel and the launch-per-block path both equal the model, through ragged sizes, a render in the middle, clone and reset.
    The mix bank runs its calls first and the per-voice twin repeats them afterwards, so that no call of the twin stops the resident kernel."""
    fn, V = RT_CASES[case]
    V = vcount(str(V))
    if too_big_for_mock(V, 1, 1200):
        pytest.skip("large for the CPU mock device")
    monkeypatch.setenv("FDSP_RT", rt)
    voices = lambda: [fn(i) for i in range(V)]   # noqa: E731
    # (bank, size, render?): bank 0 is the bank, 1 its clone
    script = [(0, s, False) for s in (64, 64, 64, 61, 8, 7, 1, 64, 33, 64, 17, 64, 64)] + [(0, 200, True)] + \
             [(0, s, False) for s in (64, 64, 64, 64, 5)] + [("clone", 0, False)] + [(0, 64, False)] * 3 + [(1, s, False) for s in (64, 64, 64, 9)] + \
             [("reset", 0, False)] + [(0, 64, False)] * 4
    banks = []

    def play(per_voice):
        b = Bank(voices(), per_voice, not per_voice)
        bs = [b]
        banks.append(b)
        rng = np.random.default_rng(11)
        nin, C = b.inputs(), b.voice_outputs()
        out = []
        for who, n, render in script:
            if who == "clone":
                bs.append(b.clone()); banks.append(bs[-1]); continue
            if who == "reset":
                b.reset(); continue
            x = rng.uniform(-1, 1, (nin, n)).astype(np.float32) if nin else None
            if render:
                r, m = bs[who].render_samples(n, x)
                out.append(r if per_voice else m)
            else:
                y = bs[who].process(n, x)
                out.append(y.reshape(V, C, n) if per_voice else y)
        return b, out

    try:
        m, mixes = play(False)
        launches = m.launch_count()
        _, rows = play(True)
        classes = bank_classes(m, voices())
        C = m.voice_outputs()
        calls = [c for c in script if c[0] not in ("clone", "reset")]
        for (who, n, render), mix, r in zip(calls, mixes, rows):
            check_mix(mix, r, classes, launch_segments(n, classes, V, C, False, False) if render else [(0, n)], False, (case, rt, who, n))
        assert max(float(np.abs(x).max()) for x in mixes) > 1e-3
        if not MOCK:   # 27 launches one per block; the resident kernel is launched about once per streak of process() calls
            assert (launches < 16) == (rt == "1"), launches
    finally:
        for b in banks:                    # destroyed here: no resident kernel outlives the test
            b.__del__()


# ---------------------------------------------------------------- stage-pipelined kernels
@pytest.mark.parametrize("staged", ["32", "128", "off"])
@pytest.mark.parametrize("name,V", [("subtractive_dry", 70), ("net", 4 * 45), ("subtractive_dry", 20)])
def test_staged_kernel_mix(name, V, staged, monkeypatch):
    """The last stage's tile at NT = 32 (HALF 16, QN 4) and 128; FDSP_STAGED=0: the plain model."""
    if MOCK and staged != "off":
        pytest.skip("the CPU mock device has no stage-pipelined form")
    monkeypatch.setenv("FDSP_STAGED", "0" if staged == "off" else "1")
    if staged != "off":
        monkeypatch.setenv("FDSP_STAGED_W", staged)
    n = 64 * 21 + 61
    inp = workloads.gate_signal(2 * n)[:, :n] if name.startswith("subtractive") else None
    mk = lambda: workloads.build(name, V)   # noqa: E731
    rows, mix, classes, segs, _ = render_and_check(mk(), n, inp, oracle=(name == "subtractive_dry"), voices_again=mk, what=(name, V, staged))
    if staged != "off" and not MOCK:
        assert any(c.stages >= 2 for c in classes)


# ---------------------------------------------------------------- multi-class banks
def test_multi_class_concurrent_streams(monkeypatch):
    """3 plain classes on the concurrent class streams (launch > 64 samples): class-order accumulate; FDSP_NO_CONCURRENT=1 gives the same bits."""
    V, n = 900, 3000 + 13
    mk = multi_voice(class_pattern(3, V, seed=9))
    voices = lambda: [mk(i) for i in range(V)]   # noqa: E731
    _, mix, *_ = render_and_check(voices(), n, voices_again=voices)
    monkeypatch.setenv("FDSP_NO_CONCURRENT", "1")
    _, mix2 = Bank(voices(), False, True).render_samples(n)
    assert np.array_equal(mix, mix2)


def test_four_class_net_bank():
    """Config 5 at its own size: 65 536 voices in 4 classes of 16 384."""
    V, n = 65536, 64 * 10
    if MOCK:
        pytest.skip("large for the CPU mock device")
    mk = lambda: workloads.build("net", V)   # noqa: E731
    rows, mix, classes, segs, _ = render_and_check(mk(), n, mix_only_too=False)
    assert len(classes) == 4
    _drop_check(rows, mix, classes, segs, False)


def test_four_class_net_bank_small():
    V, n = 4 * 33 + 2, 64 * 4 + 29
    mk = lambda: workloads.build("net", V)   # noqa: E731
    render_and_check(mk(), n, voices_again=mk)


# ---------------------------------------------------------------- two-stage (FDN) classes
@pytest.mark.parametrize("V", [33, 1024])
def test_two_stage_solo_bank(V):
    """Dry program -> FDN kernel, reduced on the second stream: the fold of its voices into a zeroed mix, across PIPE_CHUNK and TIME_CHUNK."""
    n = TIME_CHUNK + 2 * PIPE_CHUNK + 77
    if too_big_for_mock(V, 2, n):
        pytest.skip("large for the CPU mock device")
    mk = lambda: workloads.build("subtractive", V)   # noqa: E731
    _, _, classes, segs, _ = render_and_check(mk(), n, workloads.gate_signal(n), oracle=(V <= 64), voices_again=mk)
    assert is_pipelined(classes) and len(segs) >= 9


def mixed_voice(i):   # test_gpu_parity.py::test_mixed_bank_two_stage_and_plain_classes
    if i % 3 == 0:
        return workloads.subtractive_voice(i)
    if i % 3 == 1:
        return pass_() * noise().seed(i) >> lowpass_hz(400.0 + 30.0 * i, 1.0) >> pan(0.1 * (i % 7) - 0.3)
    return pass_() * saw_hz(110.0 + 5.0 * i) >> pan(-0.5)


@pytest.mark.parametrize("pipeline", ["on", "off"])
def test_two_stage_and_plain_classes(pipeline, monkeypatch):
    """Class 0 is two-stage: pipelined, the plain classes 1 and 2 add first and class 0 one chunk late; FDSP_NO_PIPELINE=1: class order."""
    if pipeline == "off":
        monkeypatch.setenv("FDSP_NO_PIPELINE", "1")
    V, n = 30, 6000 + 13
    voices = lambda: [mixed_voice(i) for i in range(V)]   # noqa: E731
    _, _, classes, _, _ = render_and_check(voices(), n, workloads.gate_signal(n), oracle=True, voices_again=voices)
    assert [c.kind for c in classes] == ["fdn_dry", "plain", "plain"] and is_pipelined(classes) == (pipeline == "on")


def reverb_input_voice(i):
    if i < 5:
        return reverb_stereo(10.0, 1.0 + 0.5 * i, 0.3 + 0.05 * i)
    return stacki(2, lambda c: pass_() * noise().seed(2 * i + c) >> lowpass_hz(500.0 + 10.0 * i, 1.0))


def test_reverb_on_bank_input():
    """reverb_stereo on the bank's stereo input: no dry program, so not pipelined; with a plain class behind it."""
    n = 5000 + 37
    rng = np.random.default_rng(3)
    x = (rng.uniform(-1, 1, (2, n)) * (np.arange(n) < 3000)).astype(np.float32)
    voices = lambda: [reverb_input_voice(i) for i in range(12)]   # noqa: E731
    _, _, classes, _, _ = render_and_check(voices(), n, x, voices_again=voices)
    assert [c.kind for c in classes] == ["fdn", "plain"] and not is_pipelined(classes)


@pytest.mark.parametrize("name", ["subtractive", "wet_only"])
def test_two_stage_process_sizes(name):
    """process(size) on a pipelined two-stage bank: zeroed, accumulated in device memory, copied out."""
    V = 9
    if name == "subtractive":
        fn = workloads.subtractive_voice
    else:
        fn = lambda i: (noise().seed(i) >> pan(0.1 * i - 0.3)) >> reverb_stereo(12.0, 1.5, 0.4)   # noqa: E731
    voices = lambda: [fn(i) for i in range(V)]   # noqa: E731
    m, t = Bank(voices(), False, True), Bank(voices(), True, False)
    classes = bank_classes(m, voices())
    assert is_pipelined(classes)
    gate = workloads.gate_signal(4000)
    at, peak = 0, 0.0
    for s in (64, 64, 17, 64, 1, 33, 64, 64, 64, 5, 64, 64) * 4:
        x = gate[:, at:at + s] if m.inputs() else None
        at += s
        mix = m.process(s, x)
        rows = t.process(s, x).reshape(V, 2, s)
        check_mix(mix, rows, classes, [(0, s)], True, (name, s))
        peak = max(peak, float(np.abs(mix).max()))
    assert peak > 1e-4


# ---------------------------------------------------------------- the device-resident entry point
def test_render_device_equals_render_samples():
    """fdsp_bank_render_device (what bench.py times) with torch CUDA buffers and a mix stride wider than n."""
    if MOCK:
        pytest.skip("torch CUDA buffers need the GPU")
    import torch
    V, n = 700, 20000 + 17
    mk = multi_voice(class_pattern(3, V, seed=2))
    voices = lambda: [mk(i) for i in range(V)]   # noqa: E731
    ref = Bank(voices(), False, True)
    _, want = ref.render_samples(n)
    b = Bank(voices(), False, True)
    stride = n + 37
    buf = torch.full((1, stride), float("nan"), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    b.render_device(n, mix_ptr=buf.data_ptr(), mix_stride=stride)
    got = buf.cpu().numpy()
    assert np.array_equal(got[:, :n], want) and np.isnan(got[:, n:]).all()
    # and the model, from a per-voice twin
    rows, _ = Bank(voices(), True, False).render_samples(n)
    classes = bank_classes(b, voices())
    check_mix(want, rows, classes, launch_segments(n, classes, V, 1, False, False), False)

"""Fill the on-disk JIT cache (fundsp_b200/jit_cache/) on a machine WITHOUT a GPU with the kernel variants the GPU test-suite uses,
so that GPU box time is not spent in NVRTC: for every graph class of tests/test_gpu_jit.py (CASES, WIDER, GATED; 40 voices each) the
layout unit and the per-voice kernel, and for the sequencer tests of tests/test_gpu_wider.py the mix variants as well. The cache is
keyed by the exact compilation (NVRTC version, options, embedded headers, source), so stale entries are never used; entries whose
headers changed can never be hit; the cache directory is emptied first (--keep: leave it). Usage: python tools/warm_jit_cache.py [-j N] [--keep]"""
import os
import sys
import time
from concurrent.futures import ProcessPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))


def has_table(sig):
    return "WaveSynth<" in sig or "PhaseSynth<" in sig


def has_heavy(sig):
    """Leaves that csrc/dsp/stage_plan.cuh gives a warp of their own (IsHeavyLeaf); when they sit on the Pipe spine the bank launches the staged kernel."""
    import re
    return "Moog<" in sig or "Dsf<" in sig or re.search(r"NlBiquad<\d+,\d+,2,", sig) is not None


def jobs():
    from fundsp_b200 import capi
    import test_gpu_jit as J
    import test_gpu_wider as W
    out = {}   # (sig, mode, tb) -> True

    def add(sig, modes):
        for m in modes:
            out[(sig, 0, 0)] = True
            for tb in ((0, 1) if has_table(sig) and m != 1 else ((1,) if has_table(sig) else (0,))):
                out[(sig, m, tb)] = True
            if has_table(sig) and m == 1:
                out[(sig, 1, 1)] = True
            if has_heavy(sig):   # the stage-pipelined kernel of the class (32 voices per CTA: what a 40-voice test bank launches), if it has one
                out[(sig, m, (1 if has_table(sig) else 0) | (32 << 8))] = True

    for table in (J.CASES, J.WIDER, J.GATED):
        for name, mk in table.items():
            for i in range(40):
                add(capi.NodeHandle(mk(i)).signature(), (1,))
    for v in W.seq_five_events().voices():
        add(capi.NodeHandle(v).signature(), (2, 3))
    for v in W.seq_loop_events(600, 44100.0).voices():                                       # test_looping_sequencer_bank_matches_oracle_sequencer (rows + mix, mix alone)
        add(capi.NodeHandle(v).signature(), (2, 3))
    from fundsp_b200.sequencer import event
    for mk in (W.live_voice, W.arp_voice):
        add(capi.NodeHandle(event(mk(100.0), 0.0, 1.0)).signature(), (2,))
    from fundsp_b200.prelude import dc, sine_hz
    add(capi.NodeHandle(event(dc(1.0), 1.0, 2.0)).signature(), (2,))
    add(capi.NodeHandle(event(sine_hz(500.0) * 0.5, 0.0, 1.0)).signature(), (2,))
    from fundsp_b200 import workloads
    from fundsp_b200.sequencer import slot
    # test_net_bank_crossfades_vertices_across_classes: the classes Xfade<old, new> the bank builds around the crossfading voices
    from fundsp_b200.prelude import noise, pass_, delay, lowpass_hz, moog_hz, pan
    sg = lambda g: capi.NodeHandle(g).signature()
    new_a = noise().seed(77) >> (pass_() & delay(0.0004)) >> lowpass_hz(700.0, 2.0) >> moog_hz(900.0, 0.3) >> pan(0.25)
    for x, y in ((workloads.net_voice(4), new_a), (workloads.net_voice(9), workloads.net_voice(22)), (new_a, workloads.net_voice(1))):
        add("Xfade<" + sg(x) + "," + sg(y) + ">", (1,))
    add(capi.NodeHandle(workloads.build("saw_svf_events", 1)[0]).signature(), (2, 3))      # bench --workload saw_svf_events and its parity test
    add(capi.NodeHandle(slot(W.arp_voice(100.0))).signature(), (1,))                        # test_slot_crossfades_to_a_new_unit
    # closures of the signal (tests/test_gpu_closures.py: rows, rows + mix; tools/bench_closures.py: mix): NVRTC-only classes
    import test_gpu_closures as CL
    from fundsp_b200.prelude import envelope2, map_, saw_hz, shape, Tanh
    for mk in CL.CASES.values():
        add(sg(mk(0)), (1, 2, 3))
    add(sg(envelope2("|t, x| x * x * a + t", a=1.0)), (1,))
    for g in (saw_hz(50.0) >> map_("|x| tanh(x[0] * drive)", 1, 1, drive=1.0), saw_hz(50.0) >> shape(Tanh(1.0))):
        add(sg(g), (1, 2, 3))
    # text envelopes (tests/test_gpu_envelope_text.py: rows, rows + mix)
    import test_gpu_envelope_text as ET
    for mk in ET.CASES.values():
        add(sg(mk(0)), (1, 2, 3))
    # the Atan and Adaptive waveshapes (tests/test_gpu_shapes.py: rows, rows + mix, the resident process() kernel of its ragged cases;
    # tools/bench_shapes.py: mix)
    import test_gpu_shapes as SH
    from fundsp_b200.prelude import Adaptive, Atan
    for mk in SH.CASES.values():
        add(sg(mk(0)), (1, 2, 3))
    for name in ("shape_atan", "shape_adaptive_4", "nlb_resonator_audio_adaptive"):
        s = sg(SH.CASES[name](0))
        out[(s, 2, (1 if has_table(s) else 0) | (255 << 8))] = True
    for g in (saw_hz(50.0) >> shape(Atan(1.0)), saw_hz(50.0) >> shape(Adaptive(0.01, Tanh(1.0)))):
        add(sg(g), (1, 2, 3))
    # prelude64: f64-state Sine and SVF classes (tests/test_gpu_prelude64.py: rows, rows + mix, the resident process() kernel of its
    # ragged cases; tools/bench_prelude64.py: mix)
    import test_gpu_prelude64 as P64
    for mk in P64.CASES.values():
        add(sg(mk(0)), (1, 2, 3))
    for name in ("sine_fm", "svf_lowpass_audio", "svf_lowshelf_hz", "headline"):
        s = sg(P64.CASES[name](0))
        out[(s, 2, (1 if has_table(s) else 0) | (255 << 8))] = True
    add(sg(saw_hz(50.0) >> lowpass_hz(1000.0, 1.0)), (1, 2, 3))
    # the exact mix model (tests/test_gpu_mix.py): 2..5-output stacks (rows, rows + mix, mix alone; twins of process() banks), the
    # 2-input stereo voice of the resident process() kernel, the plain classes beside two-stage and reverb classes
    import test_gpu_mix as MX
    for k in (2, 3, 4, 5):
        add(sg(MX.stack_voice(k)(0)), (1, 2, 3))
    for i in (1, 2):
        add(sg(MX.mixed_voice(i)), (1, 2, 3))
    add(sg(MX.reverb_input_voice(5)), (1, 2, 3))
    for name in ("in2_stereo", "five_out"):
        s = sg(MX.RT_CASES[name][0](0))
        add(s, (1, 2))
        out[(s, 2, (1 if has_table(s) else 0) | (255 << 8))] = True   # the resident process() kernel
    # the wavetable oscillators (tests/test_gpu_wavetable.py): probe voices of every kind, the mixed-kind and pipelined classes, the
    # headline class at table pitches (rows, rows + mix, mix alone, the resident process() kernel)
    import test_gpu_wavetable as WT
    for k in range(6):
        add(sg(WT.pitch_voices(k)[0][0]), (1, 2, 3))
    for v in WT.edge_bank_voices(12):
        s = sg(v)
        add(s, (1, 2, 3))
        out[(s, 2, (1 if has_table(s) else 0) | (255 << 8))] = True
    # the f32 filters (tests/test_gpu_filters.py): every audio-rate family with live and held controls (rows, the resident process()
    # kernel), at its control edges, and on both sides of a Moog stage cut (the stage-pipelined kernel at 32 and 128 voices per CTA)
    import test_gpu_filters as FL
    for fam in FL.FAM:
        for mk in (FL.live_voice, FL.held_voice, FL.edge_voice):
            s = sg(mk(fam, 0))
            add(s, (1,))
            out[(s, 2, (1 if has_table(s) else 0) | (255 << 8))] = True
        s = sg(FL.cut_voice(fam, 0))
        add(s, (1,))
        out[(s, 1, 128 << 8)] = True
    return sorted(out)


def work(job):
    from fundsp_b200 import capi
    sig, mode, tb = job
    t = time.time()
    try:
        capi.jit_precompile(sig, mode, tb)
        return job, time.time() - t, ""
    except Exception as e:   # noqa: BLE001
        return job, time.time() - t, str(e)[:300]


if __name__ == "__main__":
    n = int(sys.argv[sys.argv.index("-j") + 1]) if "-j" in sys.argv else max(1, (os.cpu_count() or 2) - 1)
    js = jobs()
    cache = os.path.join(ROOT, "fundsp_b200", "jit_cache")
    if os.path.isdir(cache) and "--keep" not in sys.argv:
        for f in os.listdir(cache):
            if f.endswith(".fdspjit") or ".tmp" in f:
                os.remove(os.path.join(cache, f))
    before = set(os.listdir(cache)) if os.path.isdir(cache) else set()
    t0 = time.time()
    bad = 0
    with ProcessPoolExecutor(n) as ex:
        for job, dt, err in ex.map(work, js, chunksize=1):
            if err:
                bad += 1
                print("FAIL", job, err)
    after = set(os.listdir(cache))
    size = sum(os.path.getsize(os.path.join(cache, f)) for f in after)
    print(f"{len(js)} units ({len(after - before)} new) in {time.time() - t0:.0f} s, cache {len(after)} files / {size / 1e6:.1f} MB, failures {bad}")
    sys.exit(1 if bad else 0)

"""Pins the oracle (and the CUDA path) to outputs of the REAL reference crate — when they exist.

`oracle/ref_dump` (a small Rust crate depending on the reference crate, fundsp 0.23.0) renders the BASELINE configurations and a few single nodes with
the real fundsp and writes tests/golden/ref/{manifest.json, *.f32}. Producing the vectors needs a Rust toolchain; until they are
committed every test below SKIPS with that reason until the directory is populated; on any machine with `cargo`
the recipe in tests/golden/ref/README.md turns "parity unpinned" (DESIGN.md §4) into a checked claim. Bar: the north-star's 1e-5
relative f32 (floor at 1e-2 of the vector's peak); the count of bit-exact samples is printed."""
import json
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "tests", "golden", "ref")
SR = 48000.0


def _manifest():
    p = os.path.join(REF, "manifest.json")
    if not os.path.exists(p):
        return None
    return json.load(open(p))


MAN = _manifest()
NAMES = [v["name"] for v in MAN["vectors"]] if MAN else ["(none)"]
need = pytest.mark.skipif(MAN is None, reason="no reference vectors: tests/golden/ref/ is empty (needs cargo and fundsp 0.23.0: oracle/ref_dump)")


def _vector(name):
    v = next(x for x in MAN["vectors"] if x["name"] == name)
    return np.fromfile(os.path.join(REF, name + ".f32"), "<f4").reshape(v["channels"], v["samples"])


def _graph(name):
    """The same graph the Rust generator built (oracle/ref_dump/src/main.rs), from the same rnd1-drawn parameters."""
    from fundsp_b200 import workloads as W
    from fundsp_b200.prelude import moog_hz, noise, reverb_stereo, saw_hz, sine_hz, white
    kind, _, idx = name.rpartition("_")
    if name == "plumbing":
        return W.plumbing(), None
    if kind == "fm":
        return W.fm_voice(int(idx)), None
    if kind == "noise_svf":
        return W.noise_svf_voice(int(idx)), None
    if kind == "saw_svf":
        return W.saw_svf_voice(int(idx)), None
    if kind == "subtractive":
        return W.subtractive_voice(int(idx)), "gate"
    return {"node_sine_440": sine_hz(440.0).phase(0.25), "node_saw_110": saw_hz(110.0).phase(0.0), "node_saw_7040": saw_hz(7040.0).phase(0.0),
            "node_moog": white().seed(1) >> moog_hz(1000.0, 0.7), "node_reverb": (white().seed(2) | white().seed(3)) >> reverb_stereo(10.0, 2.0, 0.5)}[name], None


def _gate(n):
    g = np.zeros((1, n), np.float32)
    g[0, 480:24000] = 1.0
    return g


def _close(got, want, name):
    peak = np.abs(want).max(axis=-1, keepdims=True)
    rel = np.abs(got.astype(np.float64) - want) / np.maximum(np.abs(want), 1e-2 * np.maximum(peak, 1e-30))
    print(f"{name}: {int((got == want).sum())}/{want.size} samples bit-exact, max rel err {rel.max():.3g}")
    assert rel.max() <= 1e-5, (name, float(rel.max()))


@need
@pytest.mark.parametrize("name", NAMES)
def test_oracle_matches_the_reference_crate(name):
    from oracle import OracleUnit, lib as olib
    olib().fo_set_denormal_emulation(0)
    want = _vector(name)
    g, gate = _graph(name)
    u = OracleUnit(g)
    u.set_sample_rate(SR)
    got = u.process_many(want.shape[1], _gate(want.shape[1]) if gate else None)
    _close(got, want, name)


@need
@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_gpu_matches_the_reference_crate(name):
    from fundsp_b200.bank import GpuBank
    want = _vector(name)
    g, gate = _graph(name)
    b = GpuBank([g], per_voice=True, sample_rate=SR)
    got, _ = b.render_samples(want.shape[1], _gate(want.shape[1]) if gate else None)
    _close(got[0], want, name)


def test_recipe_is_committed():
    """The generator and its instructions travel with the repository even though its output cannot be made here."""
    for p in ("oracle/ref_dump/Cargo.toml", "oracle/ref_dump/src/main.rs", "tests/golden/ref/README.md"):
        assert os.path.exists(os.path.join(ROOT, p)), p
    src = open(os.path.join(ROOT, "oracle", "ref_dump", "src", "main.rs")).read()
    for cfg in ("plumbing", "fm_", "noise_svf_", "saw_svf_", "subtractive_", "node_reverb"):
        assert cfg in src

"""The scalar-math sweep without a GPU: the committed expected hashes (tests/golden/libm_sweep.json) against a regeneration of every 16th
chunk from the oracle, the probe's NVRTC options against the closure JIT's, the probe's NVRTC build of the product's math, and the rule that
no f32 path of the product or the oracle calls the platform's trig functions (CUDA's on the device, glibc's on the host: they differ from
musl, which the reference runs, and from each other)."""
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import gen_libm_sweep  # noqa: E402

FIXTURE = os.path.join(ROOT, "tests", "golden", "libm_sweep.json")
PROBE_DIR = os.path.join(ROOT, "tools", "probe")


def _code(path):
    """The file without comments and string literals."""
    s = open(path).read()
    s = re.sub(r"/\*.*?\*/", " ", s, flags=re.S)
    s = re.sub(r"//[^\n]*", " ", s)
    return re.sub(r'"(?:\\.|[^"\\])*"', '""', s)


def test_no_platform_trig_on_f32_paths():
    files = ["fundsp_b200/csrc/dsp/libm.cuh", "fundsp_b200/csrc/dsp/math.cuh", "oracle/fo_libm.h", "oracle/fo_math.h"]
    for f in files:
        calls = re.findall(r"(?<![\w.])(?:::|std::)?(sinf|cosf|tanf|sin|cos|tan)\s*\(", _code(os.path.join(ROOT, f)))
        assert not calls, (f, calls)
    # the guard itself sees such a call
    assert re.findall(r"(?<![\w.])(?:::|std::)?(sinf|cosf|tanf|sin|cos|tan)\s*\(", "return ::sinf(x); y = std::tan(x) + k_sindf(x);") == ["sinf", "tan"]


def test_fixture_shape():
    d = json.load(open(FIXTURE))
    assert d["chunk_log2"] == 24
    want = {"sinf": 256, "cosf": 256, "tanf": 256, "tanhf": 256, "expm1f": 256, "expf": 256, "atanf": 256, "wide_sinf": 256,
            "wide_atanf": 256, "pow_x": 16, "pow_y": 16, "pow_rand": 16}
    assert {k: len(v) for k, v in d["functions"].items()} == want
    for v in d["functions"].values():
        assert all(re.fullmatch(r"[0-9a-f]{16}", h) for h in v)


def test_fixture_regenerates_every_16th_chunk(tmp_path):
    """A change to the oracle's math without a new fixture fails here, on the CPU."""
    exe = str(tmp_path / "gen_libm_sweep")
    gen_libm_sweep.build(exe)
    got = gen_libm_sweep.run(exe, every=16)["functions"]
    want = json.load(open(FIXTURE))["functions"]
    bad = [(fn, c * 16) for fn in want for c, (a, b) in enumerate(zip(got[fn], want[fn][::16])) if a != b]
    assert not bad and set(got) == set(want), bad[:20]


def _opts(path, name):
    m = re.search(r"static const char\*\s*" + name + r"\[\]\s*=\s*\{([^}]*)\}", open(path).read())
    assert m, (path, name)
    return re.findall(r'"([^"]*)"', m.group(1))


def test_probe_nvrtc_options_equal_the_jit_options():
    jit = _opts(os.path.join(ROOT, "fundsp_b200", "csrc", "host", "jit.cpp"), "kJitOpts")
    probe = _opts(os.path.join(PROBE_DIR, "libm_sweep_probe.cu"), "kJitOpts")
    assert probe == jit and "--fmad=false" in jit, (probe, jit)


def test_probe_nvrtc_build_compiles(tmp_path):
    """The probe's run-time build: the product's libm.cuh / math.cuh through NVRTC with the JIT's options (no GPU needed)."""
    exe = os.path.join(PROBE_DIR, "_build", "libm_sweep_probe")
    if not os.path.exists(exe):   # __graft_entry__.build() makes it; compile a private copy otherwise
        exe = str(tmp_path / "libm_sweep_probe")
        subprocess.check_call(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-fmad=false",
                               "-I" + os.path.join(ROOT, "fundsp_b200", "csrc", "dsp"), "-I" + os.path.join(ROOT, "tests", "golden"),
                               "-o", exe, os.path.join(PROBE_DIR, "libm_sweep_probe.cu"),
                               "-lnvrtc_static", "-lnvrtc-builtins_static", "-lnvptxcompiler_static"])
    r = subprocess.run([exe, "--root", ROOT, "--build", "nvrtc", "--compile-only"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.startswith("compiled"), r.stdout + r.stderr

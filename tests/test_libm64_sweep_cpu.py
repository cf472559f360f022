"""The f64 math sweep without a GPU, and accuracy pins of csrc/dsp/libm64.cuh and oracle/fo_libm64.h that do not come from either: the
committed expected hashes (tests/golden/libm64_sweep.json) against a regeneration of every 64th chunk from the oracle, the probe's NVRTC
options against the JIT's, the probe's NVRTC build, the rule that no f64 trig path calls the platform's functions, both tables of 2/pi and
pi/2 against mpmath, product and oracle bit for bit and within 1 ulp of mpmath at random large arguments and at the double nearest a
multiple of pi/2, and the large reduction against the medium one below their threshold."""
import ctypes as C
import json
import os
import random
import re
import struct
import subprocess
import sys

import mpmath as mp
import pytest

from oracle import lib as olib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import gen_libm64_sweep  # noqa: E402
from test_libm_sweep_cpu import _code, _opts  # noqa: E402

FIXTURE = os.path.join(ROOT, "tests", "golden", "libm64_sweep.json")
PROBE_DIR = os.path.join(ROOT, "tools", "probe")
PRODUCT = os.path.join(ROOT, "fundsp_b200", "csrc", "dsp", "libm64.cuh")
ORACLE = os.path.join(ROOT, "oracle", "fo_libm64.h")
HARD = 0x7506AC5B262CA1FF          # 6381956970095103 * 2^797, the double nearest a multiple of pi/2
THRESHOLD = 0x413921FB00000000     # the first pattern the large reduction takes: high word 0x413921fb, |x| ~ 2^20 pi/2


def d_of(u):
    return struct.unpack("<d", struct.pack("<Q", u))[0]


def b_of(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


# the trig functions of the C library and of CUDA that the guard knows by name: plain, f-suffixed, intrinsic (__sinf) and the fused or
# pi-scaled forms. A platform call through a wrapper of another name is outside what a text guard can see.
PLATFORM_TRIG = r"(?<![\w.])(?:::|std::)?(?:__)?(sin|cos|tan|sincos|sinpi|cospi|tanpi|sincospi)(?:f|l)?\s*\("


def _platform_trig_calls(code):
    """Calls of trig functions other than the files' own m64:: functions (definitions and m64::-qualified calls are removed first)."""
    code = re.sub(r"\bdouble\s+(sin|cos|tan)\s*\(\s*double\b", " ", code)
    code = re.sub(r"\bm64::(sin|cos|tan)\s*\(", " (", code)
    return re.findall(PLATFORM_TRIG, code)


def test_no_platform_trig_on_f64_paths():
    for f in (PRODUCT, ORACLE):
        calls = _platform_trig_calls(_code(f))
        assert not calls, (f, calls)
    # the guard itself sees such calls and passes the files' own
    probe = ("FDSP_HD double sin(double x) { return m64::tan(x) + ::sin(x) + std::cos(x) + tan(x) + fo::m64::cos(x) + __sinf(y) + "
             "sinpi(x) + cospif(y) + k_sin(x, y, 1); sincos(x, &s, &c); }")
    assert _platform_trig_calls(probe) == ["sin", "cos", "tan", "sin", "sinpi", "cospi", "sincos"]


def test_fixture_shape():
    d = json.load(open(FIXTURE))
    assert d["chunk_log2"] == 24
    assert {k: len(v) for k, v in d["functions"].items()} == {"sin": 514, "cos": 514, "tan": 514, "exp": 514}
    for v in d["functions"].values():
        assert all(re.fullmatch(r"[0-9a-f]{16}", h) for h in v)


def test_fixture_regenerates_every_64th_chunk_and_the_special_chunk(tmp_path):
    """A change to the oracle's f64 math or to the argument sets without a new fixture fails here, on the CPU. Chunk 513, the special
    set (rem_pio2's branch words, the large-reduction threshold, near-multiples of pi/2, exp's limits), is always regenerated."""
    exe = str(tmp_path / "gen_libm64_sweep")
    gen_libm64_sweep.build(exe)
    got = gen_libm64_sweep.run(exe, every=64, chunks=[513])["functions"]
    want = json.load(open(FIXTURE))["functions"]
    chunks = sorted(set(range(0, 514, 64)) | {513})
    assert chunks[-2:] == [512, 513]
    bad = [(fn, c) for fn in want for c, a in zip(chunks, got[fn]) if a != want[fn][c]]
    assert not bad and set(got) == set(want) and all(len(v) == len(chunks) for v in got.values()), bad[:20]


def test_probe_nvrtc_options_equal_the_jit_options():
    jit = _opts(os.path.join(ROOT, "fundsp_b200", "csrc", "host", "jit.cpp"), "kJitOpts")
    probe = _opts(os.path.join(PROBE_DIR, "libm64_sweep_probe.cu"), "kJitOpts")
    assert probe == jit and "--fmad=false" in jit, (probe, jit)


def test_probe_nvrtc_build_compiles(tmp_path):
    """The probe's run-time build: the product's libm64.cuh through NVRTC with the JIT's options (no GPU needed)."""
    exe = os.path.join(PROBE_DIR, "_build", "libm64_sweep_probe")
    if not os.path.exists(exe):   # __graft_entry__.build() makes it; compile a private copy otherwise
        exe = str(tmp_path / "libm64_sweep_probe")
        subprocess.check_call(["nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-fmad=false",
                               "-I" + os.path.join(ROOT, "fundsp_b200", "csrc", "dsp"), "-I" + os.path.join(ROOT, "tests", "golden"),
                               "-o", exe, os.path.join(PROBE_DIR, "libm64_sweep_probe.cu"),
                               "-lnvrtc_static", "-lnvrtc-builtins_static", "-lnvptxcompiler_static"])
    r = subprocess.run([exe, "--root", ROOT, "--build", "nvrtc", "--compile-only"], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.startswith("compiled"), r.stdout + r.stderr


# ---- accuracy pins against mpmath
def _two_over_pi_digits(n):
    with mp.workprec(24 * n + 64):
        f = 2 / mp.pi
        out = []
        for _ in range(n):
            f *= 2 ** 24
            v = int(mp.floor(f))
            out.append(v)
            f -= v
    return out


def _pio2_pieces(n):   # pi/2 as k_rem_pio2's PIo2[]: each piece the remainder truncated to 24 significant bits
    out = []
    with mp.workprec(400):
        r = mp.pi / 2
        for _ in range(n):
            e = int(mp.floor(mp.log(r, 2)))
            v = mp.floor(r * mp.mpf(2) ** (23 - e)) / mp.mpf(2) ** (23 - e)
            out.append(float(v))
            r -= v
    return out


def test_two_over_pi_tables_equal_mpmath():
    src = open(PRODUCT).read()
    m = re.search(r"static const int32_t ipio2\[(\d+)\] = \{([^}]*)\}", src)
    prod = [int(v, 16) for v in re.findall(r"0x([0-9A-Fa-f]+)", m.group(2))]
    assert int(m.group(1)) == len(prod) == 66
    hexs = "".join(re.findall(r'"([0-9a-f]*)"', re.search(r"TWO_OVER_PI_HEX\[\] =([^;]*);", open(ORACLE).read()).group(1)))
    orac = [int(hexs[6 * k:6 * k + 6], 16) for k in range(len(hexs) // 6)]
    assert len(hexs) == 6 * 66
    want = _two_over_pi_digits(66)
    assert prod == want and orac == want
    # the largest finite double reads digits up to jv + jk = (1000 - 3) // 24 + 4 = 45 before any recomputation
    assert (1023 - 23 - 3) // 24 + 4 == 45 < 66
    pieces = _pio2_pieces(5)
    m = re.search(r"static const uint64_t PIO2\[5\] = \{([^}]*)\}", src)
    assert [d_of(int(v, 16)) for v in re.findall(r"0x([0-9A-Fa-f]+)ull", m.group(1))] == pieces
    m = re.search(r"static const double PIo2\[5\] = \{([^}]*)\}", open(ORACLE).read())
    assert [float(v) for v in m.group(1).split(",")] == pieces


@pytest.fixture(scope="module")
def points(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("libm64") / "libm64_points")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-w", os.path.join(ROOT, "tests", "cpp", "libm64_points.cpp"), "-o", exe])

    def run(xs):
        out = subprocess.run([exe], input="".join(f"{b_of(x):016x}\n" for x in xs), capture_output=True, text=True, check=True).stdout
        rows = []
        for ln in out.splitlines():
            t = ln.split()
            row = {"sin": d_of(int(t[0], 16)), "cos": d_of(int(t[1], 16)), "tan": d_of(int(t[2], 16)),
                   "large": (int(t[3]), d_of(int(t[4], 16)), d_of(int(t[5], 16)))}
            if len(t) > 6:
                row["medium"] = (int(t[6]), d_of(int(t[7], 16)), d_of(int(t[8], 16)))
            rows.append(row)
        assert len(rows) == len(xs)
        return rows
    return run


def _oracle(fn, x):
    return {"sin": olib().fo64_sin, "cos": olib().fo64_cos, "tan": olib().fo64_tan}[fn](x)


def _ulps(got, x, fn):
    with mp.workprec(2200):
        want = {"sin": mp.sin, "cos": mp.cos, "tan": mp.tan}[fn](mp.mpf(x))
        e = int(mp.floor(mp.log(abs(want), 2)))
        ulp = mp.mpf(2) ** max(e - 52, -1074)
        return float(abs(mp.mpf(got) - want) / ulp)


def test_large_arguments_match_mpmath_and_each_other(points):
    rng = random.Random(0x6C69626D)
    xs = []
    for _ in range(3000):
        e = rng.randint(21, 1023)
        x = (1.0 + rng.random()) * 2.0 ** e
        if e == 1023:
            x = min(x, d_of(0x7FEFFFFFFFFFFFFF))
        xs.append(-x if rng.random() < 0.5 else x)
    rows = points(xs)
    worst = {"sin": 0.0, "cos": 0.0, "tan": 0.0}
    for x, row in zip(xs, rows):
        for fn in worst:
            assert b_of(row[fn]) == b_of(_oracle(fn, x)), (fn, x.hex())
            worst[fn] = max(worst[fn], _ulps(row[fn], x, fn))
    print("max ulp against mpmath over 3000 arguments of exponents 21..1023:", worst)
    assert max(worst.values()) <= 1.0, worst


def test_double_nearest_a_multiple_of_pi_over_2(points):
    x = d_of(HARD)
    with mp.workprec(2200):
        n = int(mp.nint(mp.mpf(x) / (mp.pi / 2)))
        r = mp.mpf(x) - n * (mp.pi / 2)
    assert n % 4 == 1 and abs(float(r) - 4.687165924e-19) < 1e-27
    row = points([x])[0]
    want = {"sin": 1.0, "cos": -4.6871659242546276e-19, "tan": -2.1334853857537038e18}
    for fn, w in want.items():
        for got in (row[fn], _oracle(fn, x)):
            assert _ulps(got, x, fn) <= 1.0 and abs(got - w) <= abs(w) * 2.0 ** -52, (fn, got, w)
    y = (C.c_double * 2)()
    assert olib().fo64_rem_pio2_large(x, y) % 4 == 1 and row["large"][0] % 4 == 1
    assert b_of(y[0]) == b_of(row["large"][1]) and b_of(y[1]) == b_of(row["large"][2])


def test_large_reduction_equals_medium_below_the_threshold(points):
    """Just below 2^20 pi/2 both reductions apply. k_rem_pio2's gives the n (mod 8) of e_rem_pio2's Cody-Waite steps, and both give
    x - n pi/2 as y0 + y1 to 2^-94 against mpmath. y0 alone can differ in its last bit: Cody-Waite's y0 = r - w is r - w rounded,
    not the remainder rounded, so the two agree on y0 at almost every argument but not at all."""
    rng = random.Random(7)
    us = [THRESHOLD - k for k in range(1, 2049)] + [THRESHOLD - rng.randrange(1, 1 << 40) for _ in range(2000)]
    xs = [s * d_of(u) for u in us for s in (1.0, -1.0)]
    rows = points(xs)
    y = (C.c_double * 2)()
    y0_differs = 0
    for x, row in zip(xs, rows):
        n_m, y0_m, y1_m = row["medium"]
        n_l, y0_l, y1_l = row["large"]
        assert (n_l - n_m) % 8 == 0, (x.hex(), row)
        with mp.workprec(400):
            truth = mp.mpf(x) - n_m * (mp.pi / 2)
            for y0, y1 in ((y0_l, y1_l), (y0_m, y1_m)):
                assert abs(mp.mpf(y0) + mp.mpf(y1) - truth) <= mp.mpf(2) ** -94, (x.hex(), y0, y1)
        assert abs(b_of(y0_l) - b_of(y0_m)) <= 1, x.hex()
        y0_differs += b_of(y0_l) != b_of(y0_m)
        n_o = olib().fo64_rem_pio2_large(x, y)
        assert n_o == n_l and b_of(y[0]) == b_of(y0_l) and b_of(y[1]) == b_of(y1_l), x.hex()
        n_om = olib().fo64_rem_pio2_medium(x, y)
        assert n_om == n_m and b_of(y[0]) == b_of(y0_m) and b_of(y[1]) == b_of(y1_m), x.hex()
    print(f"y0 of the two reductions differs in its last bit at {y0_differs} of {len(xs)} arguments")
    assert y0_differs <= len(xs) // 20

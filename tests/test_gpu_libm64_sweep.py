"""The product's f64 math on the H100: sin, cos, tan and exp of csrc/dsp/libm64.cuh over the three argument sets of
tests/golden/libm64_sweep_args.h (every high word with two low words, 2^24 points over the filters' domains, and the special set: rem_pio2's
branch words, the 2^20 pi/2 threshold of the large reduction, near-multiples of pi/2 up to 2^1000, exp's thresholds and the non-finite
and subnormal values). tools/probe/libm64_sweep_probe runs them in two builds of one kernel source, by nvcc with the product's flags and
by NVRTC with the JIT's options (the prelude64 nodes are built that way), and both must give the oracle's bits: the per-chunk hashes
equal tests/golden/libm64_sweep.json, which the oracle's restatement (oracle/fo_libm64.h) produces on the host."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

from oracle import lib as olib

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROBE = os.path.join(ROOT, "tools", "probe", "_build", "libm64_sweep_probe")
FIXTURE = os.path.join(ROOT, "tests", "golden", "libm64_sweep.json")
BUILDS = ("nvcc", "nvrtc")
FO_FN = {"sin": 0, "cos": 1, "tan": 2, "exp": 3}   # fo64_eval's function numbers (oracle/fo_prelude64.cpp)


def _canon(b):
    b = np.asarray(b, np.uint64).copy()
    b[(b & np.uint64(0x7FFFFFFFFFFFFFFF)) > np.uint64(0x7FF0000000000000)] = np.uint64(0x7FF8000000000000)
    return b


@pytest.fixture(scope="module")
def sweep():
    assert os.path.exists(PROBE), "tools/probe/_build/libm64_sweep_probe is missing: __graft_entry__.build() compiles it"
    res = {}
    for b in BUILDS:
        r = subprocess.run([PROBE, "--root", ROOT, "--build", b], capture_output=True, text=True, timeout=1800)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        res[b] = {d["fn"]: d for d in map(json.loads, r.stdout.splitlines())}
        for d in res[b].values():
            print(f"libm64 sweep {b:5s} {d['fn']:4s} {d['ms']:9.1f} ms")
    return res


def _first_difference(build, fn, chunk, tmp_path):
    """Argument and bits of the first result of a chunk where the device and the oracle differ."""
    out = str(tmp_path / f"{build}_{fn}_{chunk}.bin")
    r = subprocess.run([PROBE, "--root", ROOT, "--build", build, "--chunk", fn, str(chunk), out], capture_output=True, text=True, timeout=600)
    if r.returncode != 0:
        return f"(chunk dump failed: {r.stderr[-500:]})"
    d = np.fromfile(out, np.uint64).reshape(2, -1)
    x = d[0].view(np.float64).copy()
    o = np.zeros_like(x)
    P = C.POINTER(C.c_double)
    olib().fo64_eval(FO_FN[fn], x.ctypes.data_as(P), o.ctypes.data_as(P), x.size)
    bad = np.nonzero(_canon(d[1]) != _canon(o.view(np.uint64)))[0]   # past the end of the special chunk both sides are NaN
    if bad.size == 0:
        return "(the dumped chunk equals the oracle: the hash differs only through the probe's summation)"
    j = int(bad[0])
    return (f"{bad.size} results differ; first at index {(chunk << 24) + j} (x=0x{int(d[0][j]):016x} = {x[j]!r}): "
            f"device 0x{int(d[1][j]):016x}, oracle 0x{int(o.view(np.uint64)[j]):016x}")


@pytest.mark.parametrize("build", BUILDS)
def test_device_f64_math_equals_oracle(build, sweep, tmp_path):
    want = json.load(open(FIXTURE))["functions"]
    got = sweep[build]
    assert set(got) == set(want)
    bad = {fn: [c for c, (a, b) in enumerate(zip(got[fn]["hashes"], want[fn])) if a != b] for fn in want}
    bad = {fn: cs for fn, cs in bad.items() if cs}
    msg = [f"{fn}: {len(cs)} of {len(want[fn])} chunks differ (chunks {cs[:8]}...): " + _first_difference(build, fn, cs[0], tmp_path)
           for fn, cs in bad.items()]
    assert not bad, "\n".join(msg)

"""The product's scalar f32 math on the H100 over every argument: sinf cosf tanf tanhf expm1f expf atanf wide_sinf wide_atanf over all 2^32
patterns, powf over the three sets of tests/golden/libm_sweep_args.h. tools/probe/libm_sweep_probe runs them in two builds of one kernel
source, by nvcc with the product's flags and by NVRTC with the closure JIT's options, and both must give the oracle's bits: the per-chunk
hashes equal tests/golden/libm_sweep.json, which the oracle's restatements produce on the host. The same pass measures each result against
CUDA's double-precision function. Last, the fix reaches compiled closure nodes: map closures of sin, cos, tan, exp, tanh, pow and sin_hz at
edge arguments against the oracle's closure interpreter, bit for bit."""
import ctypes as C
import json
import os
import subprocess

import numpy as np
import pytest

from oracle import lib as olib, oracle_bank_render

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROBE = os.path.join(ROOT, "tools", "probe", "_build", "libm_sweep_probe")
FIXTURE = os.path.join(ROOT, "tests", "golden", "libm_sweep.json")
BUILDS = ("nvcc", "nvrtc")
# fo_libm_eval's function numbers (oracle/fundsp_oracle.cpp)
FO_FN = {"sinf": 0, "cosf": 1, "tanf": 2, "tanhf": 3, "expm1f": 4, "expf": 5, "pow_x": 6, "pow_y": 6, "pow_rand": 6, "atanf": 7,
         "wide_sinf": 8, "wide_atanf": 9}
# largest ulp error against f64 over all finite results within the f32 range (powf: normal results). wide_sinf is measured on |v| <= 2pi,
# the only domain Sine uses; its bound is the oracle's wide_sinf against glibc's f64 sin over every pattern of that domain on the host
# (1.538 ulp, at 0x4069c334 = 3.6525)
ULP_BOUND = {"sinf": 1.0, "cosf": 1.0, "expf": 1.0, "expm1f": 1.0, "tanf": 1.5, "tanhf": 2.5, "atanf": 1.0, "wide_sinf": 1.54,
             "wide_atanf": 2.85, "pow_x": 1.0, "pow_y": 1.0, "pow_rand": 1.0}


def _canon(b):
    b = np.asarray(b, np.uint32).copy()
    b[(b & 0x7FFFFFFF) > 0x7F800000] = 0x7FC00000
    return b


@pytest.fixture(scope="module")
def sweep():
    assert os.path.exists(PROBE), "tools/probe/_build/libm_sweep_probe is missing: __graft_entry__.build() compiles it"
    res = {}
    for b in BUILDS:
        r = subprocess.run([PROBE, "--root", ROOT, "--build", b], capture_output=True, text=True, timeout=1800)
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        res[b] = {d["fn"]: d for d in map(json.loads, r.stdout.splitlines())}
        for d in res[b].values():
            print(f"libm sweep {b:5s} {d['fn']:10s} {d['ms']:9.1f} ms  max ulp vs f64 {d['max_ulp']:.4f}")
    return res


def _first_difference(build, fn, chunk, tmp_path):
    """Argument and bits of the first result of a chunk where the device and the oracle differ."""
    out = str(tmp_path / f"{build}_{fn}_{chunk}.bin")
    r = subprocess.run([PROBE, "--root", ROOT, "--build", build, "--chunk", fn, str(chunk), out], capture_output=True, text=True, timeout=600)
    if r.returncode != 0:
        return f"(chunk dump failed: {r.stderr[-500:]})"
    d = np.fromfile(out, np.uint32).reshape(3, -1)
    x, y = d[0].view(np.float32).copy(), d[1].view(np.float32).copy()
    o = np.zeros_like(x)
    P = C.POINTER(C.c_float)
    olib().fo_libm_eval(FO_FN[fn], x.ctypes.data_as(P), y.ctypes.data_as(P), o.ctypes.data_as(P), x.size)
    bad = np.nonzero(_canon(d[2]) != _canon(o.view(np.uint32)))[0]
    if bad.size == 0:
        return "(the dumped chunk equals the oracle: the hash differs only through the probe's summation)"
    j = int(bad[0])
    i = (chunk << 24) + j
    arg = f"x=0x{d[0][j]:08x}" + (f", y=0x{d[1][j]:08x}" if fn.startswith("pow") else "")
    return f"{bad.size} results differ; first at index {i} ({arg}): device 0x{d[2][j]:08x}, oracle 0x{o.view(np.uint32)[j]:08x}"


@pytest.mark.parametrize("build", BUILDS)
def test_device_math_equals_oracle_over_every_argument(build, sweep, tmp_path):
    want = json.load(open(FIXTURE))["functions"]
    got = sweep[build]
    assert set(got) == set(want)
    bad = {fn: [c for c, (a, b) in enumerate(zip(got[fn]["hashes"], want[fn])) if a != b] for fn in want}
    bad = {fn: cs for fn, cs in bad.items() if cs}
    msg = [f"{fn}: {len(cs)} of {len(want[fn])} chunks differ (first chunk {cs[0]}): " + _first_difference(build, fn, cs[0], tmp_path)
           for fn, cs in bad.items()]
    assert not bad, "\n".join(msg)


def test_device_ulp_error_against_f64(sweep):
    got = sweep["nvcc"]
    over = {fn: got[fn]["max_ulp"] for fn in ULP_BOUND if not got[fn]["max_ulp"] <= ULP_BOUND[fn]}
    assert not over, (over, ULP_BOUND)
    # both builds give the same bits (test above), so the same errors
    assert all(sweep["nvrtc"][fn]["max_ulp"] == got[fn]["max_ulp"] for fn in got)


# ---- end to end: the restated functions inside compiled closure nodes

SR = 48000.0
KS = (1.0, -1.0, 0.5, 3.0)   # one voice per capture value


def _u(bits):
    return np.asarray(bits, np.uint32).view(np.float32)


def _edge_inputs():
    """Two input channels: 1024 (x, y) pairs of the powf special values, then trig and exp edges in channel 0."""
    from_x = [0x00000000, 0x80000000, 0x3F800000, 0xBF800000, 0x3F000000, 0xBF000000, 0x40000000, 0xC0000000, 0x40400000, 0xC0400000,
              0x3F800001, 0x3F7FFFFF, 0xBF800001, 0xBF7FFFFF, 0x7F800000, 0xFF800000, 0x7FC00000, 0x00000001, 0x80000001, 0x00800000,
              0x7F7FFFFF, 0xFF7FFFFF, 0x41200000, 0xC1200000, 0x3DCCCCCD, 0x3EAAAAAB, 0xC1000000, 0x40E00000, 0x3F7FBE77, 0x3F800347,
              0x0DA24260, 0x5F800000]
    from_y = [0x00000000, 0x80000000, 0x3F000000, 0xBF000000, 0x3F800000, 0xBF800000, 0x40000000, 0xC0000000, 0x40400000, 0xC0400000,
              0x3EAAAAAB, 0xBEAAAAAB, 0x4B7FFFFF, 0x4B800001, 0xCB7FFFFF, 0x4B800000, 0x7F800000, 0xFF800000, 0x7FC00000, 0x00000001,
              0x80000001, 0x3F800001, 0x3F7FFFFF, 0xBF800001, 0x3FC00000, 0xBFC00000, 0x4E000000, 0x3DCCCCCD, 0x42C80000, 0xC2C80000,
              0x42FF0000, 0xC3160000]
    px = np.repeat(np.uint32(from_x), 32)
    py = np.tile(np.uint32(from_y), 32)
    rng = np.random.default_rng(20261017)
    huge = rng.integers(0x4DC90FDB, 0x7F800000, 1500, dtype=np.uint32) | (rng.integers(0, 2, 1500, dtype=np.uint32) << 31)
    boundary = np.arange(0x4DC90FD0, 0x4DC90FE8, dtype=np.uint32)
    boundary = np.concatenate([boundary, boundary | 0x80000000])
    exp_edges = np.concatenate([np.arange(0x42B17210, 0x42B17220, dtype=np.uint32), np.arange(0x42AEAC48, 0x42AEAC58, dtype=np.uint32),
                                np.arange(0xC2CFF1B0, 0xC2CFF1BA, dtype=np.uint32), np.arange(0xC2AEAC48, 0xC2AEAC58, dtype=np.uint32),
                                np.linspace(-104.0, -87.0, 300).astype(np.float32).view(np.uint32),
                                np.linspace(-12.0, 12.0, 300).astype(np.float32).view(np.uint32)])
    specials = np.float32([0.0, -0.0, np.inf, -np.inf, np.nan, 3.4028235e38, -3.4028235e38, 1e10, -1e10, 3.5e9, 2.0**31, 1e-45,
                           np.pi, 2.0 * np.pi, 1e5, 1e7]).view(np.uint32)
    x0 = np.concatenate([px, huge, boundary, exp_edges, specials])
    x1 = np.concatenate([py, rng.uniform(-3.0, 3.0, x0.size - py.size).astype(np.float32).view(np.uint32)])
    return np.stack([_u(x0), _u(x1)])


CLOSURES = {
    "sin": "|x| sin(x[0] * k)",
    "cos": "|x| cos(x[0] * k)",
    "tan": "|x| tan(x[0] * k)",
    "exp": "|x| exp(x[0] * k)",
    "tanh": "|x| tanh(x[0] * k)",
    "pow": "|x| pow(x[0], x[1] * k)",
    "sin_hz": "|x| sin_hz(x[0], x[1] * k)",
}


@pytest.mark.parametrize("name", sorted(CLOSURES))
def test_closure_math_at_edge_arguments_matches_oracle(name):
    from fundsp_b200.bank import GpuBank
    from fundsp_b200.prelude import map_
    olib().fo_set_denormal_emulation(0)
    inp = _edge_inputs()
    n = inp.shape[1]
    mk = lambda k: map_(CLOSURES[name], 2, 1, k=k)  # noqa: E731
    b = GpuBank([mk(k) for k in KS], per_voice=True, sample_rate=SR)
    g, _ = b.render_samples(n, inp)
    o, _ = oracle_bank_render([mk(k) for k in KS], SR, n, inp)
    assert len(b.classes()) == 1
    gb, ob = _canon(g.view(np.uint32)), _canon(o.view(np.uint32))
    bad = np.argwhere(gb != ob)
    if bad.size:
        v, _, j = (int(t) for t in bad[0])
        pytest.fail(f"{name}: {len(bad)} samples differ; first voice {v} sample {j}: x = (0x{inp[0, j].view(np.uint32):08x}, "
                    f"0x{inp[1, j].view(np.uint32):08x}), device 0x{gb[v, 0, j]:08x}, oracle 0x{ob[v, 0, j]:08x}")
    assert np.isfinite(o).any() and np.isnan(o).any()

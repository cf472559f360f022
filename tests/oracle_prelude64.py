"""The oracle's prelude64 nodes (oracle/fo_prelude64.h) and f64 libm (oracle/fo_libm64.h) — TEST INFRASTRUCTURE.

They live in a library of their own, oracle/_build/libfundsp_oracle_prelude64.so, built here on first use with the flags of
oracle/Makefile. Importing this module teaches `oracle.OracleBackend` the prelude64 builders (`sine_f64`, `fixed_svf_f64`, `svf_f64`, `biquad_f64`, `butterpass_f64`, `resonator_f64`, `onepole_f64`);
they combine with every node of libfundsp_oracle.so.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import oracle

ROOT = oracle.ROOT
ODIR = os.path.join(ROOT, "oracle")
SOURCES = [os.path.join(ODIR, f) for f in ("fo_prelude64.cpp", "fo_prelude64.h", "fo_libm64.h", "fo_nodes.h", "fo_math.h", "fo_libm.h")]
CXXFLAGS = ["-O3", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-std=c++17", "-fPIC", "-fvisibility=hidden", "-pthread"]   # oracle/Makefile


def _build(out):
    os.makedirs(os.path.dirname(out), exist_ok=True)
    tmp = f"{out}.{os.getpid()}.tmp"
    subprocess.check_call(["g++", *CXXFLAGS, "-shared", "-o", tmp, SOURCES[0]])
    os.replace(tmp, out)   # atomic: concurrent test workers never load a half-written library


def build_prelude64_oracle():
    so = os.path.join(ODIR, "_build", "libfundsp_oracle_prelude64.so")
    stale = not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in SOURCES)
    if not stale:
        return so
    try:
        _build(so)
        return so
    except OSError:          # a read-only tree: build next to the process instead
        so = os.path.join(tempfile.gettempdir(), f"fdsp_oracle_prelude64_{os.getuid()}", "libfundsp_oracle_prelude64.so")
        _build(so)
        return so


_lib = None


def lib():
    global _lib
    if _lib is None:
        oracle.lib()   # the node library the prelude64 nodes are combined with
        L = C.CDLL(build_prelude64_oracle())
        P, I, F, D = C.c_void_p, C.c_int, C.c_float, C.c_double
        for name, (res, args) in {"fo64_sin": (D, [D]), "fo64_cos": (D, [D]), "fo64_tan": (D, [D]), "fo64_exp": (D, [D]),
                                  "fo_sine_f64": (P, []), "fo_fixed_svf_f64": (P, [I, F, F, F]), "fo_svf_f64": (P, [I, F, F, F]),
                                  "fo_biquad_f64": (P, [F, F, F, F, F]), "fo_butterpass_f64": (P, [F, I]), "fo_resonator_f64": (P, [F, F, I]),
                                  "fo_onepole_f64": (P, [I, F, I]), "fo_sine_f64_phase_after": (D, [C.c_uint64, D, F, I])}.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = res, args
        _lib = L
    return _lib


def _node(h):
    if not h:
        raise ValueError("the oracle has no such prelude64 node")
    return h


oracle.OracleBackend.b_sine_f64 = lambda self: _node(lib().fo_sine_f64())
oracle.OracleBackend.b_fixed_svf_f64 = lambda self, mode, f, q, g: _node(lib().fo_fixed_svf_f64(mode, f, q, g))
oracle.OracleBackend.b_svf_f64 = lambda self, mode, f, q, g: _node(lib().fo_svf_f64(mode, f, q, g))
oracle.OracleBackend.b_biquad_f64 = lambda self, a1, a2, b0, b1, b2: _node(lib().fo_biquad_f64(a1, a2, b0, b1, b2))
oracle.OracleBackend.b_butterpass_f64 = lambda self, f, nin: _node(lib().fo_butterpass_f64(f, nin))
oracle.OracleBackend.b_resonator_f64 = lambda self, f, q, nin: _node(lib().fo_resonator_f64(f, q, nin))
oracle.OracleBackend.b_onepole_f64 = lambda self, kind, p, nin: _node(lib().fo_onepole_f64(kind, p, nin))

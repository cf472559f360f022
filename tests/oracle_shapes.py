"""The oracle's Atan and Adaptive waveshapes (oracle/fo_shapes.h) — TEST INFRASTRUCTURE.

They live in a library of their own, oracle/_build/libfundsp_oracle_shapes.so, built here on first use with the flags of
oracle/Makefile. Importing this module teaches `oracle.OracleBackend` the Atan kind (6) of `shaper` and `nl_biquad` and the two
Adaptive builders; every other shape kind still goes to libfundsp_oracle.so's own Shaper and NlBiquad.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import oracle

ROOT = oracle.ROOT
ODIR = os.path.join(ROOT, "oracle")
SOURCES = [os.path.join(ODIR, f) for f in ("fo_shapes.cpp", "fo_shapes.h", "fo_nodes.h", "fo_math.h", "fo_libm.h")]
CXXFLAGS = ["-O3", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-std=c++17", "-fPIC", "-fvisibility=hidden", "-pthread"]   # oracle/Makefile


def _build(out):
    os.makedirs(os.path.dirname(out), exist_ok=True)
    tmp = f"{out}.{os.getpid()}.tmp"
    subprocess.check_call(["g++", *CXXFLAGS, "-shared", "-o", tmp, SOURCES[0]])
    os.replace(tmp, out)   # atomic: concurrent test workers never load a half-written library


def build_shapes_oracle():
    so = os.path.join(ODIR, "_build", "libfundsp_oracle_shapes.so")
    stale = not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in SOURCES)
    if not stale:
        return so
    try:
        _build(so)
        return so
    except OSError:          # a read-only tree: build next to the process instead
        so = os.path.join(tempfile.gettempdir(), f"fdsp_oracle_shapes_{os.getuid()}", "libfundsp_oracle_shapes.so")
        _build(so)
        return so


_lib = None


def lib():
    global _lib
    if _lib is None:
        oracle.lib()   # the node library the shape nodes are combined with
        L = C.CDLL(build_shapes_oracle())
        P, I, F, D = C.c_void_p, C.c_int, C.c_float, C.c_double
        for name, (res, args) in {"fo_atanf": (F, [F]), "fo_wide_atanf": (F, [F]), "fo_shaper_x": (P, [I, F, F]),
                                  "fo_shaper_adaptive": (P, [D, I, F, F]), "fo_nl_biquad_x": (P, [I, I, I, F, F, I, F, F, F]),
                                  "fo_nl_biquad_adaptive": (P, [I, I, D, I, F, F, I, F, F, F])}.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = res, args
        _lib = L
    return _lib


def _node(h):
    if not h:
        raise ValueError("the oracle has no such shape")
    return h


_b_shaper0 = oracle.OracleBackend.b_shaper
_b_nl_biquad0 = oracle.OracleBackend.b_nl_biquad


def _b_shaper(self, kind, p0, p1):
    return _node(lib().fo_shaper_x(kind, p0, p1)) if kind == 6 else _b_shaper0(self, kind, p0, p1)


def _b_nl_biquad(self, fb, mode, shape, p0, p1, nin, ce, q, g):
    return _node(lib().fo_nl_biquad_x(fb, mode, shape, p0, p1, nin, ce, q, g)) if shape == 6 else _b_nl_biquad0(self, fb, mode, shape, p0, p1, nin, ce, q, g)


def _b_shaper_adaptive(self, timescale, kind, p0, p1): return _node(lib().fo_shaper_adaptive(timescale, kind, p0, p1))
def _b_nl_biquad_adaptive(self, fb, mode, timescale, kind, p0, p1, nin, ce, q, g):
    return _node(lib().fo_nl_biquad_adaptive(fb, mode, timescale, kind, p0, p1, nin, ce, q, g))


oracle.OracleBackend.b_shaper = _b_shaper
oracle.OracleBackend.b_nl_biquad = _b_nl_biquad
oracle.OracleBackend.b_shaper_adaptive = _b_shaper_adaptive
oracle.OracleBackend.b_nl_biquad_adaptive = _b_nl_biquad_adaptive

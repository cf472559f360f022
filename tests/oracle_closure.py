"""The oracle's closure nodes (oracle/fo_closure.h: map, shape_fn, envelope_in) — TEST INFRASTRUCTURE.

They live in a library of their own, oracle/_build/libfundsp_oracle_closure.so, built here on first use with the flags of
oracle/Makefile. Importing this module teaches `oracle.OracleBackend` the three closure builders, so `OracleUnit`,
`oracle_bank_render` and everything else in tests/oracle.py lower graphs that contain closures; the closure nodes plug into the
combinators of libfundsp_oracle.so like any other oracle node.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import oracle

ROOT = oracle.ROOT
ODIR = os.path.join(ROOT, "oracle")
SOURCES = [os.path.join(ODIR, f) for f in ("fo_closure.cpp", "fo_closure.h", "fo_nodes.h", "fo_math.h", "fo_libm.h")]
CXXFLAGS = ["-O3", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-std=c++17", "-fPIC", "-fvisibility=hidden", "-pthread"]   # oracle/Makefile


def _build(out):
    os.makedirs(os.path.dirname(out), exist_ok=True)
    tmp = f"{out}.{os.getpid()}.tmp"
    subprocess.check_call(["g++", *CXXFLAGS, "-shared", "-o", tmp, SOURCES[0]])
    os.replace(tmp, out)   # atomic: concurrent test workers never load a half-written library


def build_closure_oracle():
    so = os.path.join(ODIR, "_build", "libfundsp_oracle_closure.so")
    stale = not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in SOURCES)
    if not stale:
        return so
    try:
        _build(so)
        return so
    except OSError:          # a read-only tree: build next to the process instead
        so = os.path.join(tempfile.gettempdir(), f"fdsp_oracle_closure_{os.getuid()}", "libfundsp_oracle_closure.so")
        _build(so)
        return so


_lib = None


def lib():
    global _lib
    if _lib is None:
        oracle.lib()   # the node library the closure nodes are combined with
        L = C.CDLL(build_closure_oracle())
        P, I, D, S, FP = C.c_void_p, C.c_int, C.c_double, C.c_char_p, C.POINTER(C.c_float)
        for name, args in {"fo_map": [I, I, S, I, C.POINTER(S), FP], "fo_shape_fn": [S, I, C.POINTER(S), FP],
                           "fo_envelope_in": [D, I, I, S, I, C.POINTER(S), FP]}.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = P, args
        _lib = L
    return _lib


def _caps(caps):
    names = [k.encode() for k, _ in caps]
    return len(caps), (C.c_char_p * max(1, len(caps)))(*names), (C.c_float * max(1, len(caps)))(*[v for _, v in caps])


def _node(h):
    if not h:
        raise ValueError("the oracle's closure interpreter could not parse the closure")
    return h


def _b_map(self, text, nin, nout, caps): return _node(lib().fo_map(nin, nout, text.encode(), *_caps(caps)))
def _b_shape_fn(self, text, caps): return _node(lib().fo_shape_fn(text.encode(), *_caps(caps)))
def _b_envelope_in(self, interval, text, nin, nout, caps): return _node(lib().fo_envelope_in(interval, nin, nout, text.encode(), *_caps(caps)))


oracle.OracleBackend.b_map = _b_map
oracle.OracleBackend.b_shape_fn = _b_shape_fn
oracle.OracleBackend.b_envelope_in = _b_envelope_in

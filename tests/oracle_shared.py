"""The oracle's Shared nodes (oracle/fo_shared.h: var, monitor, timer over a real shared cell) — TEST INFRASTRUCTURE.

They live in a library of their own, oracle/_build/libfundsp_oracle_shared.so, built here on first use with the flags of oracle/Makefile.
Importing this module teaches `oracle.OracleBackend` the Shared builders. Each product `Shared` gets one oracle cell of its own (its
mirror, created with the product cell's value on first use), so a test drives both sides with `set_both` and compares `s.value()` with
`mirror(s).value()`.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile
import weakref

import oracle

ROOT = oracle.ROOT
ODIR = os.path.join(ROOT, "oracle")
SOURCES = [os.path.join(ODIR, f) for f in ("fo_shared.cpp", "fo_shared.h", "fo_closure.h", "fo_nodes.h", "fo_math.h", "fo_libm.h")]
CXXFLAGS = ["-O3", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-std=c++17", "-fPIC", "-fvisibility=hidden", "-pthread"]   # oracle/Makefile


def _build(out):
    os.makedirs(os.path.dirname(out), exist_ok=True)
    tmp = f"{out}.{os.getpid()}.tmp"
    subprocess.check_call(["g++", *CXXFLAGS, "-shared", "-o", tmp, SOURCES[0]])
    os.replace(tmp, out)   # atomic: concurrent test workers never load a half-written library


def build_shared_oracle():
    so = os.path.join(ODIR, "_build", "libfundsp_oracle_shared.so")
    stale = not os.path.exists(so) or os.path.getmtime(so) < max(os.path.getmtime(s) for s in SOURCES)
    if not stale:
        return so
    try:
        _build(so)
        return so
    except OSError:          # a read-only tree: build next to the process instead
        so = os.path.join(tempfile.gettempdir(), f"fdsp_oracle_shared_{os.getuid()}", "libfundsp_oracle_shared.so")
        _build(so)
        return so


_lib = None


def lib():
    global _lib
    if _lib is None:
        oracle.lib()   # the node library the Shared nodes are combined with
        L = C.CDLL(build_shared_oracle())
        P, I, D, F = C.c_void_p, C.c_int, C.c_double, C.c_float
        for name, (res, args) in {"fo_shared_new": (P, [F]), "fo_shared_free": (None, [P]), "fo_shared_set": (None, [P, F]),
                                  "fo_shared_get": (F, [P]), "fo_var_shared": (P, [P]), "fo_monitor_shared": (P, [P, I, D]),
                                  "fo_timer": (P, [P]), "fo_var_fn": (P, [P, I, C.c_char_p, I, C.POINTER(C.c_char_p), C.POINTER(F)])}.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = res, args
        _lib = L
    return _lib


class OracleShared:
    """An oracle cell (std::shared_ptr<std::atomic<uint32_t>>)."""

    def __init__(self, value=0.0):
        self.h = lib().fo_shared_new(value)

    def set(self, v): lib().fo_shared_set(self.h, v)
    def value(self): return float(lib().fo_shared_get(self.h))

    def __del__(self):
        try:
            lib().fo_shared_free(self.h)
        except Exception:  # noqa: BLE001
            pass


_MIRRORS = weakref.WeakKeyDictionary()


def mirror(s):
    """The oracle cell that stands for the product Shared `s`."""
    m = _MIRRORS.get(s)
    if m is None:
        m = _MIRRORS[s] = OracleShared(s.value())
    return m


def set_both(s, v):
    s.set(v)
    mirror(s).set(v)


def _b_var_shared(self, s): return lib().fo_var_shared(mirror(s).h)
def _b_monitor_shared(self, s, kind, timescale): return lib().fo_monitor_shared(mirror(s).h, kind, timescale)
def _b_timer(self, s): return lib().fo_timer(mirror(s).h)


def _b_var_fn(self, s, text, nout, caps):
    names = [k.encode() for k, _ in caps]
    h = lib().fo_var_fn(mirror(s).h, nout, text.encode(), len(caps), (C.c_char_p * max(1, len(caps)))(*names),
                        (C.c_float * max(1, len(caps)))(*[v for _, v in caps]))
    if not h:
        raise ValueError("the oracle's closure interpreter could not parse the closure")
    return h


oracle.OracleBackend.b_var_shared = _b_var_shared
oracle.OracleBackend.b_monitor_shared = _b_monitor_shared
oracle.OracleBackend.b_timer = _b_timer
oracle.OracleBackend.b_var_fn = _b_var_fn

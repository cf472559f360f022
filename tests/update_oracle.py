"""The oracle's System<X, F> for the tests of `update` (tests/cpp/oracle_system.cpp) — TEST INFRASTRUCTURE.

`split_update` reads an update text on its own (not with the product's parser): its parameters, its `let`s and each `x.set(..)`
statement's setting, arguments and address. `fos_system` runs the arguments through the oracle's closure interpreter and applies the
settings through the oracle nodes' set(). `oracle_of(expr)` is `expr` as the oracle builds it, with every `update` as that System.
"""
import ctypes as C
import os
import re
import subprocess
import tempfile

from oracle import OracleBackend, _caps, _node, lib as olib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "oracle_system.cpp")
KINDS = {"center": 1, "center_q": 2, "center_q_gain": 3, "value": 4, "biquad": 6, "pan": 11}

_lib = None


def lib():
    global _lib
    if _lib is None:
        olib()
        d = os.path.join(tempfile.gettempdir(), f"fdsp_oracle_system_{os.getuid()}")
        os.makedirs(d, exist_ok=True)
        deps = [SRC] + [os.path.join(ROOT, "oracle", f) for f in os.listdir(os.path.join(ROOT, "oracle")) if f.startswith("fo_") and f.endswith(".h")]
        so = os.path.join(d, f"liboracle_system_{int(max(os.path.getmtime(p) for p in deps))}.so")
        if not os.path.exists(so):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.check_call(["g++", "-O2", "-march=x86-64-v3", "-ffp-contract=off", "-fno-fast-math", "-std=c++17", "-fPIC", "-shared",
                                   "-fvisibility=hidden", "-w", SRC, "-o", tmp])
            os.replace(tmp, so)
        L = C.CDLL(so)
        I, P = C.c_int, C.c_void_p
        L.fos_system.restype = P
        L.fos_system.argtypes = [P, C.c_float, C.c_char_p, I, C.POINTER(C.c_char_p), C.POINTER(C.c_float), I, C.POINTER(I), C.POINTER(I),
                                 C.POINTER(I), C.POINTER(C.c_int64)]
        _lib = L
    return _lib


def _top(s, sep):
    """Split `s` at `sep` outside brackets."""
    out, depth, cur = [], 0, ""
    for ch in s:
        if ch in "([{":
            depth += 1
        elif ch in ")]}":
            depth -= 1
        if ch == sep and depth == 0:
            out.append(cur)
            cur = ""
        else:
            cur += ch
    out.append(cur)
    return out


def split_update(text):
    """(t name, dt name, [let statements], [(kind, [argument texts], [address])])"""
    m = re.match(r"\s*(?:move\s+)?\|([^|]*)\|", text)
    names = [p.split(":")[0].strip() for p in m.group(1).split(",")]
    body = text[m.end():].strip()
    if body.startswith("{"):
        body = body[1:-1]
    lets, sets = [], []
    for st in (x.strip() for x in _top(body, ";")):
        if not st:
            continue
        if st.startswith("let "):
            lets.append(st + ";")
            continue
        h = re.match(r"(\w+)\s*\.\s*set\s*\(\s*Setting\s*::\s*(\w+)\s*\(", st)
        assert h and h.group(1) == names[2], st
        depth, i = 1, h.end()
        while depth:
            depth += {"(": 1, ")": -1}.get(st[i], 0)
            i += 1
        args = [a.strip() for a in _top(st[h.end():i - 1], ",") if a.strip()]
        address = [0 if k == "left" else 1 if k == "right" else int(n) for k, n in re.findall(r"\.\s*(left|right|index)\s*\(\s*(\d*)\s*\)", st[i:])]
        sets.append((KINDS[h.group(2)], args, address))
    return names[0], names[1], lets, sets


def system(x, dt, text, caps):
    """An oracle System around the oracle node x (consumed)."""
    t, d, lets, sets = split_update(text)
    args = [a for _, a_, _ in sets for a in a_]
    value = args[0] if len(args) == 1 else "(" + ", ".join(args) + ")"
    fn = f"|{t}, {d}, __unused| {{ {' '.join(lets)} {value} }}"
    I = C.c_int
    kinds = (I * len(sets))(*[k for k, _, _ in sets])
    nargs = (I * len(sets))(*[len(a) for _, a, _ in sets])
    naddr = (I * len(sets))(*[len(ad) for _, _, ad in sets])
    flat = [v for _, _, ad in sets for v in ad]
    addr = (C.c_int64 * max(1, len(flat)))(*flat)
    return _node(lib().fos_system(x, dt, fn.encode(), *_caps(caps), len(sets), kinds, nargs, naddr, addr))


class _WithUpdate:
    """The oracle backend, with `update` lowered as the System above."""

    def __init__(self, be):
        self.be = be

    def __getattr__(self, name):
        return getattr(self.be, name)

    def b_update(self, dt, text, caps, x): return system(x, dt, text, caps)
    def b_netnode(self, net): return net.lower(self)
    def b_seqnode(self, seq): return seq.lower(self)


class oracle_of:
    """`expr` as the oracle builds it: OracleUnit and oracle_bank_render take it in place of the expression."""

    def __init__(self, expr):
        self.expr = expr

    def lower(self, be):
        return self.expr.lower(_WithUpdate(be if isinstance(be, OracleBackend) else OracleBackend()))

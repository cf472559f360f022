"""fundsp_b200 — H100-native block-processing engine for FunDSP's voice-bank hot path.

`prelude` mirrors the reference's opcode vocabulary, `graph.An` its operators; `GpuBank` evaluates V voice
instances on the GPU through the C ABI in include/fundsp_b200.h (libfundsp_b200.so, hand-written sm_90a CUDA).
"""
from . import prelude  # noqa: F401
from .graph import An, ArityError  # noqa: F401


def __getattr__(name):  # lazy: importing the package must not require the shared library
    if name in ("GpuBank", "FdspError"):
        from . import bank
        return getattr(bank, name)
    raise AttributeError(name)

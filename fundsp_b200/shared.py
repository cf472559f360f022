"""Shared controls (src/shared.rs:47-81): a float that any thread sets and reads, and that graphs read with `var(s)` and write with
`monitor(s, meter)` and `timer(s)`.

A `Shared` is a 32-bit cell in host memory, read and written with relaxed atomics like the reference's `Arc<AtomicU32>`. Every node
built on it, and every bank that holds such a node, keeps its own reference, so the cell lives as long as any of them.

A bank reads its readers' cells once before each `process()` / `render` call, so a value set between two calls holds from the first
sample of the next call to its end. After a call it stores into each written cell what the last writer in processing order stores: the
last voice in bank order, and within that voice the last writer in evaluation order.
"""
from __future__ import annotations

from . import capi
from .graph import f32


class Shared:
    """Shared::new(value): `set` / `set_value` store a value, `value` reads it."""

    __slots__ = ("handle", "__weakref__")

    def __init__(self, value=0.0):
        self.handle = capi.lib().fdsp_shared_new(f32(value))
        if not self.handle:
            raise MemoryError("fdsp_shared_new")

    def set(self, value):
        capi.lib().fdsp_shared_set(self.handle, f32(value))

    set_value = set

    def value(self):
        return float(capi.lib().fdsp_shared_get(self.handle))

    def __del__(self):
        try:
            if self.handle:
                capi.lib().fdsp_shared_free(self.handle)
                self.handle = None
        except Exception:  # noqa: BLE001  (interpreter shutdown)
            pass

    def __repr__(self):
        return f"Shared({self.value()!r})"


def shared(value=0.0):
    """shared(value) (src/prelude.rs): a new Shared."""
    return Shared(value)

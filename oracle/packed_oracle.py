"""TEST INFRASTRUCTURE ONLY -- numpy oracle of packed destinations in direct weight sync.

The element rule, restated on whole global arrays: each element of a packed destination inside part p's
box, at local index i, takes the value of source ``p.source`` at global index
``p.source_offsets + (i - box start)``, with the int-indexed dims dropped first.  Elements outside every
part keep what they held.  Parts are read by attribute (``source``, ``dest_index``, ``source_offsets``),
so this module shares no code with the package.
"""

from __future__ import annotations

import numpy as np


def fill(dest: np.ndarray, parts, sources: dict) -> np.ndarray:
    """A copy of ``dest`` with every part applied; ``sources`` maps source names to their global arrays."""
    out = dest.copy()
    for p in parts:
        box = out[p.dest_index]
        src = sources[p.source]
        window = tuple(slice(o, o + e) for o, e in zip(p.source_offsets, box.shape))
        assert len(window) == src.ndim, "a part's box has the rank of its source"
        out[p.dest_index] = src[window]
    return out


def shard(global_array: np.ndarray, offsets, shape) -> np.ndarray:
    """The shard of ``global_array`` at ``offsets`` with ``shape`` (what an unpacked TP destination holds)."""
    return global_array[tuple(slice(o, o + e) for o, e in zip(offsets, shape))].copy()


def destination(layout_entry, sources: dict, name: str, fill_value=0, dtype=None) -> np.ndarray:
    """The expected content of one destination of a generator layout entry ``(local shape, parts, box)``:
    the parts applied to a ``fill_value`` array, or the shard of the same-named source when ``parts`` is None."""
    shape, parts, box = layout_entry
    if parts is None:
        return shard(sources[name], box[0], shape)
    dt = dtype if dtype is not None else next(iter(sources[p.source] for p in parts)).dtype
    return fill(np.full(shape, fill_value, dtype=dt), parts, sources)

"""TEST INFRASTRUCTURE ONLY -- numpy oracle of transposed packed parts in direct weight sync.

A packed part with ``transpose = True`` fills a box that, with its int-indexed dims dropped, has shape
``(..., a, b)`` from the source box of shape ``(..., b, a)`` at ``source_offsets`` (source coordinates): box
element ``(..., i, j)`` takes source element ``source_offsets + (..., j, i)``.  Restated on whole arrays, the box
receives ``src_box.swapaxes(-1, -2)``; equivalently it reads ``src.swapaxes(-1, -2)`` at the offsets with their last
two entries swapped.  Parts are read by attribute (``source``, ``dest_index``, ``source_offsets``, ``transpose``),
so this module shares no code with the package.
"""

from __future__ import annotations

from dataclasses import dataclass

import numpy as np


def read(src: np.ndarray, offsets, box_shape) -> np.ndarray:
    """What a transposed part with a box of ``box_shape`` (int dims dropped) reads from ``src`` at ``offsets``, element
    by element: ``out[..., i, j] = src[offsets + (..., j, i)]``."""
    out = np.empty(box_shape, dtype=src.dtype)
    for idx in np.ndindex(*box_shape):
        s = idx[:-2] + (idx[-1], idx[-2])
        out[idx] = src[tuple(o + x for o, x in zip(offsets, s))]
    return out


def fill(dest: np.ndarray, parts, sources: dict) -> np.ndarray:
    """A copy of ``dest`` with every part applied (transposed parts swapped); ``sources`` maps source names to their
    global arrays."""
    out = dest.copy()
    for p in parts:
        box = out[p.dest_index]
        src = sources[p.source]
        ext = box.shape[:-2] + box.shape[:-3:-1] if getattr(p, "transpose", False) else box.shape
        window = tuple(slice(o, o + e) for o, e in zip(p.source_offsets, ext))
        assert len(window) == src.ndim, "a part's box has the rank of its source"
        out[p.dest_index] = src[window].swapaxes(-1, -2) if getattr(p, "transpose", False) else src[window]
    return out


@dataclass(frozen=True)
class Part:
    """An untransposed part, for the other oracles' ``fill``."""

    source: str
    dest_index: tuple
    source_offsets: tuple


def plain(parts, sources: dict) -> tuple[list, dict]:
    """The same fill without transposed parts: ``(parts, sources)`` where every transposed part reads a transposed
    copy of its whole source at its offsets with the last two swapped.  ``packed_oracle.fill`` of the result, or any
    oracle that fills from whole sources, then equals ``fill``.  Sources may be any per-element arrays."""
    out_parts, out_sources = [], dict(sources)
    for p in parts:
        offs = tuple(p.source_offsets)
        if not getattr(p, "transpose", False):
            out_parts.append(Part(p.source, p.dest_index, offs))
            continue
        name = f"{p.source}#T"
        if name not in out_sources:
            out_sources[name] = np.ascontiguousarray(sources[p.source].swapaxes(-1, -2))
        out_parts.append(Part(name, p.dest_index, offs[:-2] + (offs[-1], offs[-2])))
    return out_parts, out_sources


def destination(layout_entry, sources: dict, name: str, fill_value=0, dtype=None) -> np.ndarray:
    """The expected content of one destination of a generator layout entry ``(local shape, parts, box)``: the parts
    applied to a ``fill_value`` array, or the shard of the same-named source when ``parts`` is None."""
    shape, parts, box = layout_entry
    if parts is None:
        return sources[name][tuple(slice(o, o + e) for o, e in zip(box[0], shape))].copy()
    dt = dtype if dtype is not None else sources[parts[0].source].dtype
    return fill(np.full(shape, fill_value, dtype=dt), parts, sources)

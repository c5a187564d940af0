"""TEST INFRASTRUCTURE ONLY -- numpy oracle of rotary packed parts in direct weight sync.

A packed part with ``rotary_head_dim = hd`` reads a source whose heads (``hd`` rows each along dim -2, the first
at source row 0) hold their rows in interleaved rotary order, pairs ``(2j, 2j + 1)`` (Meta / torchtitan), and fills
its box in half-split order, pairs ``(j, j + hd / 2)`` (Hugging Face / vLLM): box row ``h * hd + t * hd / 2 + j``
takes source row ``source_offsets[-2] + h * hd + 2 * j + t``.  Restated on whole arrays, the box receives
``src_box.reshape(lead + (H, hd / 2, 2, C)).swapaxes(-3, -2).reshape(lead + (H * hd, C))``.  Parts are read by
attribute (``source``, ``dest_index``, ``source_offsets``, ``rotary_head_dim``), so this module shares no code with
the package.
"""

from __future__ import annotations

from dataclasses import dataclass

import numpy as np


def half_split(a: np.ndarray, hd: int) -> np.ndarray:
    """``a`` with the rows (axis -2) of every ``hd``-row head moved from interleaved into half-split order."""
    lead, (rows, cols) = a.shape[:-2], a.shape[-2:]
    assert rows % hd == 0 and hd % 2 == 0
    return a.reshape(lead + (rows // hd, hd // 2, 2, cols)).swapaxes(-3, -2).reshape(a.shape)


def fill(dest: np.ndarray, parts, sources: dict) -> np.ndarray:
    """A copy of ``dest`` with every part applied (rotary parts reordered); ``sources`` maps source names to their
    global arrays."""
    out = dest.copy()
    for p in parts:
        box = out[p.dest_index]
        window = tuple(slice(o, o + e) for o, e in zip(p.source_offsets, box.shape))
        assert len(window) == sources[p.source].ndim, "a part's box has the rank of its source"
        src = sources[p.source][window]
        hd = getattr(p, "rotary_head_dim", None)
        out[p.dest_index] = src if hd is None else half_split(src, hd)
    return out


@dataclass(frozen=True)
class Part:
    """A part without a rotary order, for the other oracles' ``fill``."""

    source: str
    dest_index: tuple
    source_offsets: tuple


def plain(parts, sources: dict) -> tuple[list, dict]:
    """The same fill without rotary parts: ``(parts, sources)`` where every rotary part reads, at the same offsets,
    a half-split copy of its whole source (heads start at source row 0).  ``packed_oracle.fill`` of the result, or
    any oracle that fills from whole sources, then equals ``fill``.  Sources may be any per-element arrays (values,
    dequantised values, ...)."""
    out_parts, out_sources = [], dict(sources)
    for p in parts:
        hd = getattr(p, "rotary_head_dim", None)
        if hd is None:
            out_parts.append(Part(p.source, p.dest_index, tuple(p.source_offsets)))
            continue
        name = f"{p.source}#half_split{hd}"
        if name not in out_sources:
            out_sources[name] = half_split(sources[p.source], hd)
        out_parts.append(Part(name, p.dest_index, tuple(p.source_offsets)))
    return out_parts, out_sources


def destination(layout_entry, sources: dict, name: str, fill_value=0, dtype=None) -> np.ndarray:
    """The expected content of one destination of a generator layout entry ``(local shape, parts, box)``: the parts
    applied to a ``fill_value`` array, or the shard of the same-named source when ``parts`` is None."""
    shape, parts, box = layout_entry
    if parts is None:
        return sources[name][tuple(slice(o, o + e) for o, e in zip(box[0], shape))].copy()
    dt = dtype if dtype is not None else sources[parts[0].source].dtype
    return fill(np.full(shape, fill_value, dtype=dt), parts, sources)

"""TEST INFRASTRUCTURE ONLY -- reference of the verbatim pull (scaled float8_e4m3fn sources moved as they are into
a scaled float8_e4m3fn destination of the same granularity).

``verbatim`` works group by group on numpy arrays and shares no code with the package's mapping.  Source shards
are ``(q, scale, offset)``: e4m3fn bytes of the shard, its float32 scale as published (the groups the shard
touches, anchored at the global origin) and its global offset in every dim.  The destination is a box
``(offset, shape)``.

* Replicated shards: a shard whose part of the destination equals an earlier shard's part is skipped, as the
  planner reads each region once.  Every destination element must then be covered exactly once (ValueError).
* Destination groups are anchored at the destination's local origin: 128x128 blocks, one row per channel, the
  [rows, cols] matrix per tensor, each leading index on its own.  Source groups are anchored at the global
  origin and cut by their shard.
* Walking the destination groups in lexicographic order ``lead + (group row, group col)``, the first group
  whose elements lie in two shards or in two source groups is returned.  Otherwise every destination byte is
  the source byte at the same global index and every destination scale the source scale of the group that
  holds it.
"""

from __future__ import annotations

import itertools

import numpy as np

BLOCK = 128


def group_size(granularity: str, rows: int, cols: int) -> tuple[int, int]:
    """(rows, cols) of a destination group of a [rows, cols] matrix (edge blocks are cut by the matrix)."""
    return {"block": (BLOCK, BLOCK), "channel": (1, cols), "tensor": (rows, cols)}[granularity]


def scale_grid(granularity: str, scale: np.ndarray, shape, r0: int, c0: int) -> np.ndarray:
    """A published scale viewed as ``lead + (group rows, group cols)`` of a ``shape`` shard at (r0, c0)."""
    *lead, n, k = shape
    if granularity == "block":
        grid = (-(-(r0 + n) // BLOCK) - r0 // BLOCK, -(-(c0 + k) // BLOCK) - c0 // BLOCK)
    else:
        grid = (n, 1) if granularity == "channel" else (1, 1)
    return np.asarray(scale, np.float32).reshape(tuple(lead) + grid)


def source_group(granularity: str, row: int, col: int) -> tuple[int, int]:
    """The global source group (row, col) of global element (row, col) of one leading index."""
    return {"block": (row // BLOCK, col // BLOCK), "channel": (row, 0), "tensor": (0, 0)}[granularity]


def verbatim(granularity: str, sources: list, offset, shape):
    """-> ``(q uint8 [shape], scale float32 lead + (group rows, group cols), None)``, or ``(None, None, group)``
    with the first destination group that does not lie inside one source group of one shard."""
    box = [(o, o + e) for o, e in zip(offset, shape)]
    kept, regions = [], set()
    for q, s, off in sources:
        region = tuple((max(o, b0), min(o + e, b1)) for o, e, (b0, b1) in zip(off, q.shape, box))
        if any(a >= b for a, b in region) or region in regions:
            continue
        regions.add(region)
        kept.append((q, s, off, region))
    owner = np.full(shape, -1, np.int64)
    count = np.zeros(shape, np.int64)
    for i, (_, _, _, region) in enumerate(kept):
        idx = tuple(slice(a - o, b - o) for (a, b), o in zip(region, offset))
        owner[idx] = i
        count[idx] += 1
    if not (count == 1).all():
        raise ValueError(f"{int((count == 0).sum())} elements covered by no shard, {int((count > 1).sum())} by two")
    *lead, n, k = shape
    gr, gc = group_size(granularity, n, k)
    n_gr, n_gc = -(-n // gr), -(-k // gc)
    out_q = np.zeros(shape, np.uint8)
    out_s = np.zeros(tuple(lead) + (n_gr, n_gc), np.float32)
    for b in itertools.product(*(range(e) for e in lead)):
        for i, j in itertools.product(range(n_gr), range(n_gc)):
            rows = range(i * gr, min((i + 1) * gr, n))
            cols = range(j * gc, min((j + 1) * gc, k))
            owners = np.unique(owner[b + (slice(rows.start, rows.stop), slice(cols.start, cols.stop))])
            groups = {source_group(granularity, offset[-2] + r, offset[-1] + c) for r in (rows[0], rows[-1])
                      for c in (cols[0], cols[-1])}  # groups are boxes: the corners hold every one
            if len(owners) != 1 or len(groups) != 1:
                return None, None, b + (i, j)
            q, s, off, _ = kept[int(owners[0])]
            grid = scale_grid(granularity, s, q.shape, off[-2], off[-1])
            sr, sc = groups.pop()
            r0g, c0g = source_group(granularity, off[-2], off[-1])
            src_b = tuple(x + o - so for x, o, so in zip(b, offset[:-2], off[:-2]))
            out_s[b + (i, j)] = grid[src_b + (sr - r0g, sc - c0g)]
    for q, _, off, region in kept:
        out_q[tuple(slice(a - o, b - o) for (a, b), o in zip(region, offset))] = \
            q[tuple(slice(a - o, b - o) for (a, b), o in zip(region, off))]
    return out_q, out_s, None

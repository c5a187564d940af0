"""Edge-biased workloads for copy_rects' plain fp8 casts (float8_e4m3fn, float8_e5m2 <-> f32, bf16,
f16), shared by tests/test_fp8_cast_regimes_cpu.py and tests/test_gpu_fp8_cast_regimes.py.

The windows are those of tests/helpers.edge_case, aimed at the kernel's tile boundaries, but sized in
the fp8 vector unit: 16 elements (64 or 32 bytes on the wide side, one 16-byte access on the fp8
side), not the 8 of the 16-bit casts.  Every base is allocated with one tile of the widest unit
behind it, so a mover that runs past a row's end lands in bytes the comparison covers."""

from __future__ import annotations

import random

import numpy as np
import torch

from tests.helpers import (EDGE_KINDS, RectCase, _edge_outer, _edge_window, edge_geometry, edge_workload,
                           random_bits)
from tests.test_fp8_cast_cpu import FP8_PAIRS, VECTOR_MODE

E4M3 = torch.float8_e4m3fn
FP8_EPU = 16  # elements per vector unit of every fp8 cast
TILE_UNITS = (64, 256, 4096, 32768)  # the tile sizes of the regime matrix (1, 4, 64 and 512 KiB tiles)
WORKLOADS = ("fp8", "bf16_e4m3", "fp8_mixed")
PINNED_KINDS = ("wide_remainder", "narrow_nd_tiles")
# kinds a scalar window is drawn with: the geometric ones (a scalar unit is one element)
SCALAR_KINDS = tuple(k for k in EDGE_KINDS if k not in ("aligned", "cast_vector"))
SLACK_BYTES = 64  # per tile unit: the widest unit (16 f32 elements)
GUARD = 0xA5


def _geometry(rng: random.Random, tile_units: int, kind: str):
    """(units per row, rows, outer dims) of `kind`: helpers.edge_geometry, plus two kinds that reach
    their regime whatever the draw.  wide_remainder: a wide row of one or two whole tiles and a short
    last segment.  narrow_nd_tiles: narrow rows of more than one tile under two outer dims (an even row
    count, which helpers._edge_outer always splits in two)."""
    T = tile_units
    if kind == "wide_remainder":
        return rng.choice([1, 2]) * T + rng.choice([1, 7, T // 2, T - 1]), rng.choice([1, 2, 3]), rng.choice([0, 1, 2])
    if kind == "narrow_nd_tiles":
        units = rng.choice([1, 3, T // 3, T - 1])
        split = T // units
        return units, 2 * max(2, split // 2 + rng.randint(1, max(1, split // 2))), 2
    return edge_geometry(rng, T, kind)


def fp8_edge_case(rng: random.Random, tile_units: int, kind: str, pair, vector: bool | None = None) -> RectCase:
    """One window of `kind` (helpers.EDGE_KINDS, wide_remainder or narrow_nd_tiles) casting pair =
    (src dtype, dst dtype), one of test_fp8_cast_cpu.FP8_PAIRS, for copy tiles of `tile_units` units.

    vector=True: 16-byte aligned windows whose rows are whole 16-element units (a vector mode);
    vector=False: windows one element off alignment (the scalar mode); None: cast_vector and aligned
    are vector, cast_scalar is scalar, any other kind is either with even odds."""
    sdt, ddt = pair
    if vector is None:
        vector = kind != "cast_scalar" and (kind in ("aligned", "cast_vector") or rng.random() < 0.5)
    units, rows, n_outer = _geometry(rng, tile_units, kind)
    outer = _edge_outer(rng, rows, n_outer) if n_outer else []
    if not outer and rows > 1:
        outer = [rows]
    shape = outer + [units * (FP8_EPU if vector else 1)]
    pad_outer = kind in ("wide_nd", "deep_nd", "narrow_nd_tiles") or rng.random() < 0.7  # padded: outer dims never merge
    sbase, sidx = _edge_window(rng, shape, sdt.itemsize, vector, pad_outer)
    dbase, didx = _edge_window(rng, shape, ddt.itemsize, vector, pad_outer)
    if not vector:
        if rng.random() < 0.5:
            dbase, didx = _edge_window(rng, shape, ddt.itemsize, True, pad_outer)  # one clean side
        # the outer starts can bring a window one element off back onto 16 bytes: step the source off again
        # (its base has at least one spare element after the window's row)
        offset = np.ravel_multi_index([s.start for s in sidx], sbase) * sdt.itemsize
        if offset % 16 == 0:
            sidx = sidx[:-1] + (slice(sidx[-1].start + 1, sidx[-1].stop + 1),)
    return RectCase(sbase, dbase, sdt, ddt, lambda b, i=sidx: b[i], lambda b, i=didx: b[i])


def fp8_edge_workload(rng: random.Random, tile_units: int, uniform: str | None = None, mixed: bool = False) -> list:
    """Edge windows of every fp8 mode for copy tiles of `tile_units` units, shuffled.

    Default: for each of the 12 pairs a vector wide_remainder row, a vector narrow_nd_tiles window and
    a scalar window of a geometric edge kind, then every edge kind once more on a drawn pair: all 24
    fp8 modes.  uniform="bf16_e4m3": every edge kind and both pinned kinds as vector bf16->e4m3 windows
    only, so the plan compiles to KIND_BF16_E4M3.  mixed=True: the default windows plus
    helpers.edge_workload's byte moves and 16-bit casts, one KIND_GENERIC plan whose 16-byte moves take
    link tiles under TSB_LINK=2."""
    T = tile_units
    if uniform == "bf16_e4m3":
        kinds = [k for k in EDGE_KINDS if k != "cast_scalar"] + list(PINNED_KINDS) * 2
        return [fp8_edge_case(rng, T, k, (torch.bfloat16, E4M3), vector=True) for k in kinds]
    assert uniform is None, uniform
    cases = []
    for i, pair in enumerate(FP8_PAIRS):
        cases += [fp8_edge_case(rng, T, k, pair, vector=True) for k in PINNED_KINDS]
        cases.append(fp8_edge_case(rng, T, SCALAR_KINDS[i % len(SCALAR_KINDS)], pair, vector=False))
    cases += [fp8_edge_case(rng, T, k, rng.choice(FP8_PAIRS)) for k in EDGE_KINDS]
    if mixed:
        cases += edge_workload(rng, T, extra=0)
    rng.shuffle(cases)
    return cases


def workload(name: str, tile_units: int) -> list:
    """The seeded cases of one workload of WORKLOADS at one tile size: the GPU and CPU files draw the same."""
    rng = random.Random(f"fp8-regimes-{tile_units}-{name}")
    if name == "bf16_e4m3":
        return fp8_edge_workload(rng, tile_units, uniform="bf16_e4m3")
    return fp8_edge_workload(rng, tile_units, mixed=name == "fp8_mixed")


def materialise(cases, device, seed: int, tile_units: int):
    """Like helpers.materialise, but each base is the front of a flat allocation with one tile of the
    widest unit behind it: zeros behind a source, GUARD bytes behind a destination.  Returns
    [(src_view, dst_view, dst_alloc, src_alloc)]; the allocations are 1-D and the comparisons cover all
    of dst_alloc."""
    gen = torch.Generator().manual_seed(seed)
    slack = SLACK_BYTES * tile_units
    out = []
    for c in cases:
        ns, nd = int(np.prod(c.src_base_shape)), int(np.prod(c.dst_base_shape))
        src = torch.cat([random_bits((ns,), c.src_dtype, gen), torch.zeros(slack // c.src_dtype.itemsize, dtype=c.src_dtype)])
        finite = c.dst_dtype.itemsize > 1  # torch has no isfinite for fp8; their bytes are compared exactly
        dst = torch.cat([random_bits((nd,), c.dst_dtype, gen, finite).view(torch.uint8),
                         torch.full((slack,), GUARD, dtype=torch.uint8)]).view(c.dst_dtype)
        src, dst = src.to(device), dst.to(device)
        out.append((c.src_view(src[:ns].view(c.src_base_shape)), dst_window(c, dst), dst, src))
    return out


def dst_window(case: RectCase, alloc: torch.Tensor) -> torch.Tensor:
    """The destination window of `case` inside a destination allocation of materialise (or a clone)."""
    return case.dst_view(alloc[: int(np.prod(case.dst_base_shape))].view(case.dst_base_shape))


# ---- what the compiled tables must reach ----------------------------------------------------------------
FP8_VECTOR_MODES = tuple(sorted(VECTOR_MODE.values()))
FP8_MODES = tuple(m for v in FP8_VECTOR_MODES for m in (v, v + 1))


def mode_regimes(fields: np.ndarray, tile_units: int) -> dict:
    """mode -> the fp8 mover regimes its copy-queue rects reach: a wide row whose last segment is short,
    a wide row of two or more tiles, a narrow N-D rect, and one that spans several tiles."""
    f = fields[fields["tile_units"] == tile_units]
    out = {}
    for m in sorted(set(f["mode"].tolist()) & set(FP8_MODES)):
        g = f[f["mode"] == m]
        wide, upr, rows, split = (g[k].astype(np.int64) for k in ("wide", "units_per_row", "rows", "split"))
        nd = (wide == 0) & (g["n_outer"] >= 2)
        out[m] = {
            "wide_remainder": bool(((wide == 1) & (upr % tile_units != 0)).any()),
            "wide_multi_tile": bool(((wide == 1) & (split >= 2)).any()),
            "narrow_nd": bool(nd.any()),
            "narrow_nd_multi_tile": bool((nd & (rows > split)).any()),
        }
    return out

"""Named branches of the quantising pulls (csrc/block_fp8.cu and csrc/scaled_fp8.cu), decided from the compiled
tables.

Every regime is a predicate over the record arrays ``_native.block_fp8_compile_host`` (blocks, pieces) and
``_native.scaled_fp8_compile_host`` (bands, pieces, tiles, n_groups) return for one pull, plus the geometry of
its destinations and source shards, and names the workload that reaches it.  A workload is one
``DirectWeightSyncDest.pull``: one or more names, each a global bf16/f16/f32 tensor cut into source shards
(optionally starting some elements past a 16-byte boundary), one destination window and a granularity.  The
names of one pull share one block plan and one per-channel / per-tensor plan per device.  The CPU suite
compiles every workload on host memory through the planner and replays it against the oracles; the H100 suite
pulls it and asserts the regime again from the tables of the live plan's inputs.

Branches:
  block_fp8_kernel   one 256-thread CTA per 128x128 block (edge blocks partial), of any target of the plan; the
                     dynamic stage is sized by the plan's widest source dtype (64 KiB when any block is f32) and
                     each block switches on its own src_dtype.  Its pieces land in the stage in source dtype:
                     ``vec`` pieces (source, stride and width 16-byte aligned, and (col0 * es) % 16 == 0) take
                     16-byte loads, the others load element by element (a 4-byte branch for f32, a 2-byte one
                     widening bf16 or f16).  The block's |x| max is one CTA reduction; the stage is then narrowed
                     16 elements per thread and step, one 16-byte store when the destination row is 16-byte
                     aligned (pitch % 16 == 0) and the chunk whole, byte stores otherwise.
  scaled_fp8_rows_kernel
                     per-channel rows of at most 32 KiB: bands of at most min(256, 32768 / round16(cols * es))
                     whole rows of one matrix, one CTA each; one s_amax and one s_scale word per band row (all 256
                     in a 256-row band).  In stage_band a warp step is 32 lanes x 4 16-byte units (vec pieces) or
                     32 elements (byte pieces); a step inside one row is warp-reduced and written by one lane, a
                     step that spans rows takes a per-lane atomicMax.  Pieces off a 16-byte column of the row are
                     byte-wise; the stage pitch is padded to 16 bytes.
  two-pass tiles     per-tensor matrices and per-channel rows over 32 KiB: tiles of at most 16384 elements of one
                     source box, one amax word per group (atomicMax, cleared before pass 1), the tile at (row 0,
                     column 0) of its group writes scale_inv; ``vec`` when the tile's source is 16-byte aligned.
"""

from __future__ import annotations

import random
from collections import defaultdict
from dataclasses import dataclass
from typing import Callable

import numpy as np
import torch

from oracle import block_fp8_oracle, int8_source_oracle, scaled_fp8_oracle, ue8m0_oracle
from oracle.block_fp8_oracle import synth_f32
from tests.fp8_regimes import draw, split, whole
from tests.helpers import (DEV, E4M3, KW, assert_same_bits_or_nan, dest_scale_shape, guarded, guards_intact, named,
                           rand_full, region, run)
from tests.source_quant_regimes import on_device
from tests.test_block_fp8_cpu import assert_block_fp8_equal
from tests.test_scaled_fp8_cpu import assert_scaled_fp8_equal
from torchstore_b200 import _native
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource
from torchstore_b200.transport.types import TensorSlice
from torchstore_b200.planner import build_rects

BLOCK, STAGE_BYTES, TILE_ELEMS, BAND_ROWS = 128, 32768, 16384, 256
VEC_STEP_UNITS, BYTE_STEP_ELEMS = 32 * 4, 32  # one warp step of stage_band: 32 lanes x kUnroll 16-byte units, or 32 elements
ES = {"bfloat16": 2, "float16": 2, "float32": 4}
CODE = {"bfloat16": _native.TSB_BF16, "float16": _native.TSB_F16, "float32": _native.TSB_F32}
NAME = {v: k for k, v in CODE.items()}
GRANULARITIES = ("block", "channel", "tensor")


@dataclass(frozen=True)
class Pull:
    """One quantised name of a workload."""
    dtype: str         # source dtype of every shard: "bfloat16", "float16" or "float32"
    shape: tuple       # global shape [..., N, K]
    src: tuple         # source shards: ((offset, local shape), ...)
    dst: tuple         # destination window: (offset, local shape)
    g: str             # "block", "channel" or "tensor"
    misalign: tuple = ()  # per source shard: its first element this many elements past a 16-byte boundary

    def shift(self, r: int) -> int:
        return self.misalign[r] if r < len(self.misalign) else 0

    def describe(self) -> str:
        mis = f" misalign={list(self.misalign)}" if any(self.misalign) else ""
        return f"{self.g} {self.dtype}{list(self.shape)} src={list(self.src)}{mis} dst={self.dst}"


@dataclass(frozen=True)
class Workload:
    pulls: tuple  # of Pull, the names w0, w1, ... of one pull
    seed: int

    def describe(self) -> str:
        return "; ".join(f"w{i}: {p.describe()}" for i, p in enumerate(self.pulls))


def cut(shape, dim: int, bounds) -> tuple:
    """Shards of `shape` along `dim` at the given boundaries (0 and the end implied)."""
    edges = [0, *bounds, shape[dim]]
    out = []
    for a, b in zip(edges, edges[1:]):
        off, loc = [0] * len(shape), list(shape)
        off[dim], loc[dim] = a, b - a
        out.append((tuple(off), tuple(loc)))
    return tuple(out)


def mesh(rows, cols) -> tuple:
    """The intersections of row shards and column shards of one shape."""
    return tuple((ro[:-1] + (co[-1],), rl[:-1] + (cl[-1],)) for ro, rl in rows for co, cl in cols)


def _p(dtype, shape, src=None, g="block", dst=None, misalign=()):
    return Pull(dtype, tuple(shape), tuple(src or (whole(shape),)), dst or whole(shape), g, tuple(misalign))


def _w(seed, *pulls):
    return Workload(tuple(pulls), seed)


WORKLOADS: dict[str, Workload] = {
    # block plans
    **{f"blk_aligned_{d}": _w(1 + i, _p(d, (256, 384), split((256, 384), 2, 0))) for i, d in enumerate(ES)},
    **{f"blk_misaligned_{d}": _w(4 + i, _p(d, (130, 260), misalign=(1,))) for i, d in enumerate(ES)},
    # 8 row shards x columns [0, 40) (80-byte rows: vec), [40, 136) (vec) and [136, 300) (328-byte rows: byte-wise);
    # 300-byte destination rows
    "blk_many_pieces": _w(7, _p("bfloat16", (256, 300), mesh(split((256, 300), 8, 0), cut((256, 300), 1, (40, 136))))),
    # columns [4, 124): 240-byte aligned rows that start 8 bytes into the block's first 16-byte column
    "blk_off_column": _w(8, _p("float16", (256, 388), cut((256, 388), 1, (4, 124)))),
    "blk_narrow": _w(9, _p("bfloat16", (200, 12), split((200, 12), 3, 0))),
    "blk_one_row": _w(10, _p("float32", (257, 200), split((257, 200), 2, 0))),
    "blk_stack_corner": _w(11, _p("bfloat16", (3, 130, 260), split((3, 130, 260), 3, 1))),
    "blk_replicas": _w(12, _p("bfloat16", (256, 200), split((256, 200), 2, 0) * 2, dst=split((256, 200), 2, 1)[1])),
    "blk_mixed_dtypes": _w(13, _p("bfloat16", (256, 260), split((256, 260), 3, 0)),
                           _p("float32", (130, 200), split((130, 200), 2, 1)),
                           _p("float16", (200, 136), misalign=(1,))),
    # per-channel bands
    "ch_tall_bf16": _w(20, _p("bfloat16", (600, 64), cut((600, 64), 1, (32,)), "channel")),
    "ch_tall_f32": _w(21, _p("float32", (520, 32), cut((520, 32), 1, (16,)), "channel")),
    "ch_band_204_rows": _w(22, _p("float16", (400, 80), g="channel")),
    "ch_rows_of_128_units": _w(23, _p("bfloat16", (64, 1024), split((64, 1024), 2, 0), "channel")),
    "ch_rows_of_200_units": _w(24, _p("float16", (40, 1600), g="channel")),
    "ch_byte_narrow": _w(25, _p("float32", (300, 20), g="channel", misalign=(1,))),
    "ch_byte_rows_of_320": _w(26, _p("bfloat16", (100, 320), g="channel", misalign=(1,))),
    "ch_byte_rows_of_100": _w(27, _p("float16", (100, 100), g="channel", misalign=(1,))),
    "ch_col_shards": _w(28, _p("bfloat16", (256, 260), split((256, 260), 2, 1), "channel")),
    "ch_stage_bound_bfloat16": _w(29, _p("bfloat16", (3, 16384), g="channel")),
    "ch_stage_bound_float16": _w(30, _p("float16", (3, 16384), split((3, 16384), 3, 1), "channel")),
    "ch_stage_bound_float32": _w(31, _p("float32", (3, 8192), split((3, 8192), 2, 1), "channel")),
    "ch_stack": _w(32, _p("float32", (3, 130, 48), split((3, 130, 48), 3, 0), "channel")),
    # two-pass tiles
    "tn_aligned_stack": _w(40, _p("bfloat16", (2, 256, 512), split((2, 256, 512), 2, 1), "tensor")),
    "tn_misaligned": _w(41, _p("float16", (300, 260), g="tensor", misalign=(1,))),
    "tn_mesh": _w(42, _p("float32", (300, 260), mesh(split((300, 260), 2, 0), split((300, 260), 3, 1)), "tensor")),
    "ch_long_col_shards": _w(43, _p("bfloat16", (4, 16400), split((4, 16400), 3, 1), "channel")),
    "tn_long_rows": _w(44, _p("float16", (3, 40000), g="tensor")),
    "tn_many_matrices": _w(45, _p("bfloat16", (300, 16, 64), split((300, 16, 64), 2, 0), "tensor")),
    # bands of two dtypes and tiles of two dtypes in one plan
    "scaled_mixed": _w(46, _p("bfloat16", (200, 96), split((200, 96), 2, 0), "channel"),
                       _p("float32", (130, 72), g="channel"),
                       _p("float16", (2, 64, 200), split((2, 64, 200), 2, 1), "tensor"),
                       _p("bfloat16", (300, 260), split((300, 260), 2, 1), "tensor")),
}


# ---- the tables of one pull ------------------------------------------------------------------------
@dataclass
class Tables:
    block: tuple | None   # (blocks, pieces) of the block plan
    scaled: tuple | None  # (bands, pieces, tiles, n_groups) of the per-channel / per-tensor plan


@dataclass(frozen=True)
class Dest:
    ptr: int
    batch: int
    rows: int
    cols: int
    g: str


@dataclass(frozen=True)
class Source:
    lo: int
    hi: int
    pull: int     # index of its name in the workload
    off: tuple    # global offset and local shape of the shard
    loc: tuple
    es: int


@dataclass(frozen=True)
class Geometry:
    """What a predicate may know besides the tables: the fp8 destinations and every source shard."""
    dests: tuple
    sources: tuple

    def dest_of(self, addr: int) -> Dest:
        return next(d for d in self.dests if d.ptr <= addr < d.ptr + d.batch * d.rows * d.cols)

    def matrix_of(self, addr: int) -> int:
        d = self.dest_of(addr)
        return (addr - d.ptr) // (d.rows * d.cols)

    def row_of(self, addr: int) -> int:
        d = self.dest_of(addr)
        return (addr - d.ptr) % (d.rows * d.cols) // d.cols

    def col_of(self, addr: int) -> int:
        d = self.dest_of(addr)
        return (addr - d.ptr) % d.cols

    def source_of(self, addr: int) -> int:
        return next(i for i, s in enumerate(self.sources) if s.lo <= addr < s.hi)

    def coord(self, addr: int) -> tuple[int, tuple]:
        """(name index, global coordinate) of the source element at byte `addr`."""
        s = self.sources[self.source_of(addr)]
        local = np.unravel_index((addr - s.lo) // s.es, s.loc)
        return s.pull, tuple(int(o + i) for o, i in zip(s.off, local))


def compile_tables(pulls, ops, handles, window_of, dests, scales, flags: int = 0) -> tuple[Tables, Geometry]:
    """Compile on the host the quantising plans a pull of `pulls` (names w0, w1, ...) builds: the windows of
    `ops` (the planner's ops of the pull, the quantised names' ones used) with `window_of(buffer)` mapping a
    source buffer, and the targets of the fp8 (or int8) destinations `dests` and their `scales`, in the order the pull
    orders them (block, channel, tensor names), with the plan `flags` (0 or _native.TSB_QUANT_UE8M0).  -> (Tables,
    Geometry); keep `dests`, `scales` alive."""
    grans = {f"w{i}": p.g for i, p in enumerate(pulls)}
    order = sorted(grans, key=lambda n: GRANULARITIES.index(grans[n]))
    pairs = {True: [], False: []}
    for op in ops:
        if op.name in grans:
            pairs[grans[op.name] == "block"].append(DirectWeightSyncDest.op_windows(op, window_of(op.rdma_buffer)))
    tables = Tables(None, None)
    for block in (True, False):
        names = [n for n in order if (grans[n] == "block") == block]
        if not names:
            continue
        rects, nr = build_rects(pairs[block], quantise=True)  # TSB_I8 rects for int8 destinations
        arr = _native.make_target_array(len(names)) if block else _native.make_sq_target_array(len(names))
        for i, n in enumerate(names):
            d, s = dests[n], scales[n]
            rows, cols = d.shape[-2:]
            args = (d.data_ptr(), s.data_ptr(), d.numel() // (rows * cols), rows, cols)
            arr[i] = _native.BqTarget(*args) if block else \
                _native.SqTarget(*args, _native.TSB_SCALE_PER_CHANNEL if grans[n] == "channel" else _native.TSB_SCALE_PER_TENSOR, 0)
        if block:
            tables.block = _native.block_fp8_compile_host(0, rects, nr, arr, len(names), flags)
        else:
            tables.scaled = _native.scaled_fp8_compile_host(0, rects, nr, arr, len(names), flags)
    dgeom = []
    for n in order:
        d = dests[n]
        rows, cols = d.shape[-2:]
        dgeom.append(Dest(d.data_ptr(), d.numel() // (rows * cols), rows, cols, grans[n]))
    sgeom = []
    for i, p in enumerate(pulls):
        for h in handles[f"w{i}"]:
            m = window_of(h.rdma_buffer)
            n = int(np.prod(m.shape, dtype=np.int64))
            sgeom.append(Source(m.ptr, m.ptr + n * ES[p.dtype], i, tuple(h.tensor_slice.offsets),
                                tuple(h.tensor_slice.local_shape), ES[p.dtype]))
    return tables, Geometry(tuple(dgeom), tuple(sgeom))


def plan_bytes(tables: Tables) -> dict:
    """{"block" / "scaled": (CTAs of pass 1, source bytes read)}: what plan_info reports as num_tiles and src_bytes."""
    out = {}
    if tables.block is not None:
        blocks, pieces = tables.block
        es = np.array([ES[NAME[int(b["src_dtype"])]] for b in blocks for _ in range(int(b["n_pieces"]))], dtype=np.int64)
        out["block"] = (len(blocks), int((pieces["rows"].astype(np.int64) * pieces["cols"] * es).sum()) if len(pieces) else 0)
    if tables.scaled is not None:
        bands, pieces, tiles, _ = tables.scaled
        es = np.array([ES[NAME[int(b["src_dtype"])]] for b in bands for _ in range(int(b["n_pieces"]))], dtype=np.int64)
        read = int((pieces["rows"].astype(np.int64) * pieces["cols"] * es).sum()) if len(pieces) else 0
        tes = np.array([ES[NAME[int(d)]] for d in tiles["src_dtype"]], dtype=np.int64)
        read += int((tiles["rows"].astype(np.int64) * tiles["cols"] * tes).sum()) if len(tiles) else 0
        out["scaled"] = (len(bands) + len(tiles), read)
    return out


# ---- predicates ----------------------------------------------------------------------------------
def _with_pieces(units, pieces):
    return [(u, pieces[int(u["piece0"]): int(u["piece0"]) + int(u["n_pieces"])]) for u in units]


def blocks_of(tb: Tables):
    return _with_pieces(*tb.block) if tb.block is not None else []


def bands_of(tb: Tables):
    return _with_pieces(*tb.scaled[:2]) if tb.scaled is not None else []


def tiles_of(tb: Tables):
    return tb.scaled[2] if tb.scaled is not None else []


def es_of(u) -> int:
    return ES[NAME[int(u["src_dtype"])]]


def _block(f):
    return lambda tb, g: any(f(b, ps, g) for b, ps in blocks_of(tb))


def _band(f):
    return lambda tb, g: any(f(b, ps, g) for b, ps in bands_of(tb))


def _band_piece(f):
    """A piece of a band of more than one row, given (piece, element size)."""
    return _band(lambda b, ps, g: int(b["rows"]) > 1 and any(f(p, es_of(b)) for p in ps))


def units_per_row(p, es) -> int:
    return int(p["cols"]) * es // 16


def aligned_source(p, es) -> bool:
    """Source, stride and width 16-byte aligned: the piece is byte-wise only because of its column."""
    return int(p["src"]) % 16 == 0 and (int(p["rows"]) == 1 or int(p["src_stride"]) % 16 == 0) and int(p["cols"]) * es % 16 == 0


def read_once(tb, g) -> bool:
    """Replicated shards among the sources, the pieces reading each destination element from one of them."""
    read = sum(int(p["rows"]) * int(p["cols"]) * es_of(b) for b, ps in blocks_of(tb) for p in ps)
    want = sum(int(b["rows"]) * int(b["cols"]) * es_of(b) for b, _ in blocks_of(tb))
    used = {g.source_of(int(p["src"])) for _, ps in blocks_of(tb) for p in ps}
    offsets = [(s.off, s.loc) for s in g.sources]
    return read == want and len(set(offsets)) < len(offsets) and len(used) == len(set(offsets))


def groups_of(tiles, g, gran):
    """{group: its tiles} of the tiles whose destination has granularity `gran`."""
    out = defaultdict(list)
    for t in tiles:
        if g.dest_of(int(t["dst"])).g == gran:
            out[int(t["group"])].append(t)
    return out


def one_writer_at_origin(ts, g, gran) -> bool:
    """Exactly one tile of the group writes scale_inv: the one at column 0 (and row 0 of the matrix per tensor)."""
    w = [t for t in ts if int(t["scale_inv"])]
    return len(w) == 1 and g.col_of(int(w[0]["dst"])) == 0 and (gran == "channel" or g.row_of(int(w[0]["dst"])) == 0)


def tensor_group_over_mesh(tb, g) -> bool:
    groups = groups_of(tiles_of(tb), g, "tensor")
    return bool(groups) and all(one_writer_at_origin(ts, g, "tensor") for ts in groups.values()) and any(
        len({g.col_of(int(t["dst"])) for t in ts}) > 1 and len({g.row_of(int(t["dst"])) for t in ts}) > 1
        and len({g.source_of(int(t["src"])) for t in ts}) >= 4 for ts in groups.values())


def channel_rows_over_stage(tb, g) -> bool:
    groups = groups_of(tiles_of(tb), g, "channel")
    return bool(groups) and not bands_of(tb) and all(
        one_writer_at_origin(ts, g, "channel") and len({g.source_of(int(t["src"])) for t in ts}) > 1 for ts in groups.values())


def one_writer_per_group(tb) -> bool:
    tiles, n = tiles_of(tb), tb.scaled[3] if tb.scaled is not None else 0
    return len(tiles) > 0 and (tiles["scale_inv"] != 0).sum() == n and len({int(t["group"]) for t in tiles if int(t["scale_inv"])}) == n


@dataclass(frozen=True)
class Regime:
    workload: str
    holds: Callable  # (Tables, Geometry) -> bool
    doc: str


REGIMES: dict[str, Regime] = {
    # block_fp8_kernel
    **{f"block_all_vec_{d}": Regime(f"blk_aligned_{d}",
                                    _block(lambda b, ps, g, d=d: NAME[int(b["src_dtype"])] == d and (ps["vec"] == 1).all()
                                           and int(b["rows"]) == BLOCK and int(b["cols"]) == BLOCK),
                                    f"{d} 128x128 block whose pieces all take 16-byte loads")
       for d in ES},
    **{f"block_byte_piece_{d}": Regime(f"blk_misaligned_{d}",
                                       _block(lambda b, ps, g, d=d: NAME[int(b["src_dtype"])] == d and (ps["vec"] == 0).any()),
                                       f"{d} block with a piece loaded element by element")
       for d in ES},
    "block_vec_and_byte_pieces": Regime("blk_many_pieces", _block(lambda b, ps, g: (ps["vec"] == 1).any() and (ps["vec"] == 0).any()),
                                        "block assembled from 16-byte and byte-wise pieces"),
    "block_of_8_pieces": Regime("blk_many_pieces", _block(lambda b, ps, g: len(ps) >= 8),
                                "block assembled from 8 or more pieces of a row x column mesh"),
    "block_pitch_off_16": Regime("blk_many_pieces", _block(lambda b, ps, g: int(b["pitch"]) % 16 != 0 and int(b["cols"]) >= 16),
                                 "block of whole 16-column chunks in rows that are not 16-byte aligned (byte stores)"),
    "block_piece_off_16_columns": Regime(
        "blk_off_column", _block(lambda b, ps, g: any(int(p["vec"]) == 0 and aligned_source(p, es_of(b))
                                                      and int(p["col0"]) * es_of(b) % 16 != 0 for p in ps)),
        "f16 piece with an aligned source and stride that starts off a 16-byte column of the block"),
    "block_under_16_columns": Regime("blk_narrow", _block(lambda b, ps, g: int(b["cols"]) < 16),
                                     "block of 12 columns: one partial 16-element chunk per row"),
    "block_one_row": Regime("blk_one_row", _block(lambda b, ps, g: int(b["rows"]) == 1),
                            "f32 block of one row"),
    "block_partial_corner_in_stack": Regime(
        "blk_stack_corner", _block(lambda b, ps, g: int(b["rows"]) < BLOCK and int(b["cols"]) < BLOCK and g.matrix_of(int(b["dst"])) > 0),
        "block partial in rows and columns in a matrix past the first of a stack"),
    "block_mixed_dtypes": Regime("blk_mixed_dtypes",
                                 lambda tb, g: {"bfloat16", "float32"} <= {NAME[int(b["src_dtype"])] for b, _ in blocks_of(tb)},
                                 "one block plan of bf16, f16 and f32 blocks: a 64 KiB stage under 2-byte blocks"),
    "block_replica_read_once": Regime("blk_replicas", read_once, "replicated source shards, each byte read once"),
    # scaled_fp8_rows_kernel
    **{f"band_256_rows_{d}": Regime(f"ch_tall_{'bf16' if d == 'bfloat16' else 'f32'}",
                                    _band(lambda b, ps, g, d=d: int(b["rows"]) == BAND_ROWS and NAME[int(b["src_dtype"])] == d),
                                    f"{d} band of 256 rows: every s_amax and s_scale word")
       for d in ("bfloat16", "float32")},
    "band_129_to_255_rows": Regime("ch_band_204_rows", _band(lambda b, ps, g: 128 < int(b["rows"]) < BAND_ROWS),
                                   "band of more than 128 and fewer than 256 rows"),
    "band_vec_steps_span_rows": Regime("ch_tall_bf16", _band_piece(lambda p, es: int(p["vec"]) == 1 and units_per_row(p, es) < VEC_STEP_UNITS),
                                       "vec piece of rows under 128 units: every warp step spans rows (per-lane atomicMax)"),
    "band_vec_steps_in_one_row": Regime(
        "ch_rows_of_128_units", _band_piece(lambda p, es: int(p["vec"]) == 1 and units_per_row(p, es) % VEC_STEP_UNITS == 0),
        "vec piece of rows of 128 units: every warp step in one row (warp-reduced, one lane writes)"),
    "band_vec_steps_mixed": Regime(
        "ch_rows_of_200_units", _band_piece(lambda p, es: int(p["vec"]) == 1 and units_per_row(p, es) > VEC_STEP_UNITS
                                            and units_per_row(p, es) % VEC_STEP_UNITS != 0),
        "vec piece of rows of 200 units: warp steps inside one row and across two"),
    "band_byte_steps_span_rows": Regime("ch_byte_narrow", _band_piece(lambda p, es: int(p["vec"]) == 0 and int(p["cols"]) < BYTE_STEP_ELEMS),
                                        "byte piece of rows under 32 elements: every warp step spans rows"),
    "band_byte_steps_in_one_row": Regime(
        "ch_byte_rows_of_320", _band_piece(lambda p, es: int(p["vec"]) == 0 and int(p["cols"]) % BYTE_STEP_ELEMS == 0),
        "byte piece of rows of a multiple of 32 elements: every warp step in one row"),
    "band_byte_steps_mixed": Regime(
        "ch_byte_rows_of_100", _band_piece(lambda p, es: int(p["vec"]) == 0 and int(p["cols"]) > BYTE_STEP_ELEMS
                                           and int(p["cols"]) % BYTE_STEP_ELEMS != 0),
        "byte piece of rows of 100 elements: warp steps inside one row and across two"),
    "band_piece_off_16_columns": Regime("ch_col_shards", _band(lambda b, ps, g: len(ps) > 1 and (ps["col0"] * es_of(b) % 16 != 0).any()),
                                        "band of column shards, one starting off a 16-byte column"),
    "band_padded_stage_pitch": Regime("ch_col_shards", _band(lambda b, ps, g: int(b["rows"]) > 1 and int(b["cols"]) * es_of(b) % 16 != 0),
                                      "band of 520-byte rows: the stage pitch is padded to 528"),
    **{f"band_one_row_at_stage_bound_{d}": Regime(
        f"ch_stage_bound_{d}", _band(lambda b, ps, g, d=d: int(b["rows"]) == 1 and int(b["cols"]) * ES[d] == STAGE_BYTES
                                     and NAME[int(b["src_dtype"])] == d),
        f"{d} band of one row of exactly 32 KiB")
       for d in ES},
    "band_in_stack": Regime("ch_stack", _band(lambda b, ps, g: g.matrix_of(int(b["dst"])) > 0),
                            "band of a matrix past the first of a stack"),
    "band_mixed_dtypes": Regime("scaled_mixed", lambda tb, g: len({int(b["src_dtype"]) for b, _ in bands_of(tb)}) > 1,
                                "bands of bf16 and f32 rows in one launch"),
    # two-pass tiles
    "tile_tensor_rows_vec": Regime("tn_aligned_stack", lambda tb, g: any(int(t["rows"]) > 1 and int(t["vec"]) == 1 for t in tiles_of(tb)),
                                   "per-tensor tile of several rows, 16-byte loads"),
    "tile_tensor_rows_byte": Regime("tn_misaligned", lambda tb, g: any(int(t["rows"]) > 1 and int(t["vec"]) == 0 for t in tiles_of(tb)),
                                    "per-tensor tile of several rows, element-wise loads"),
    "tile_tensor_group_over_mesh": Regime("tn_mesh", tensor_group_over_mesh,
                                          "per-tensor group of tiles over two row ranges and three column shards, one scale_inv "
                                          "writer at (0, 0)"),
    "tile_channel_rows_over_stage": Regime("ch_long_col_shards", channel_rows_over_stage,
                                           "per-channel rows over 32 KiB from column shards: one group per row, its writer at column 0"),
    "tile_full_width_and_remainder": Regime(
        "tn_long_rows", lambda tb, g: any(int(t["cols"]) == TILE_ELEMS for t in tiles_of(tb)) and any(
            0 < int(t["cols"]) < TILE_ELEMS and g.col_of(int(t["dst"])) > 0 and g.col_of(int(t["dst"])) % TILE_ELEMS == 0
            for t in tiles_of(tb)),
        "16384-column tiles and the remainder tile of a row"),
    "tile_over_256_groups": Regime("tn_many_matrices", lambda tb, g: tb.scaled is not None and tb.scaled[3] > 256 and one_writer_per_group(tb),
                                   "per-tensor stack of 300 matrices: more than 256 amax words"),
    "bands_and_tiles": Regime("scaled_mixed", lambda tb, g: len(bands_of(tb)) > 0 and len(tiles_of(tb)) > 0,
                              "channel bands and tensor tiles in one plan"),
}


# ---- places a slip would show ----------------------------------------------------------------------
def _step_ends(p, es):
    """(first element, last element) of every warp step of a band piece, as piece-local (row, column)."""
    rows, cols = int(p["rows"]), int(p["cols"])
    if int(p["vec"]):
        per, upr = 16 // es, units_per_row(p, es)
        total, step = rows * upr, VEC_STEP_UNITS
        first = lambda u: (u // upr, u % upr * per)  # noqa: E731
        last = lambda u: (u // upr, u % upr * per + per - 1)  # noqa: E731
    else:
        total, step = rows * cols, BYTE_STEP_ELEMS
        first = last = lambda e: (e // cols, e % cols)  # noqa: E731
    for s in range(0, total, step):
        yield first(s), last(min(s + step, total) - 1)


def spots(tables: Tables, geom: Geometry, cap: int = 32) -> dict[int, list]:
    """{name index: global coordinates} where the kernels branch: the first and the last lane of the first and
    the last warp step of each band piece that spans rows, then the first and the last element of every piece
    (byte-wise pieces off a 16-byte column first), then of every tile.  At most `cap` per name."""
    out = defaultdict(list)

    def add(p, es, rc):
        i, c = geom.coord(int(p["src"]) + rc[0] * int(p["src_stride"]) + rc[1] * es)
        if c not in out[i]:
            out[i].append(c)

    for b, ps in bands_of(tables):
        for p in ps:
            span = [(f, l) for f, l in _step_ends(p, es_of(b)) if f[0] != l[0]]
            for f, l in span[:1] + span[-1:]:
                add(p, es_of(b), f)
                add(p, es_of(b), l)
    pieces = [(p, es_of(u)) for u, ps in blocks_of(tables) + bands_of(tables) for p in ps]
    pieces.sort(key=lambda x: (int(x[0]["vec"]), int(x[0]["col0"]) * x[1] % 16 == 0))
    for p, es in pieces:
        add(p, es, (0, 0))
        add(p, es, (int(p["rows"]) - 1, int(p["cols"]) - 1))
    for t in tiles_of(tables):
        es = es_of(t)
        add(t, es, (0, 0))
        add(t, es, (int(t["rows"]) - 1, int(t["cols"]) - 1))
    return {i: (c if len(c) <= cap else c[: cap // 2] + c[-(cap // 2):]) for i, c in out.items()}


# ---- on the H100 ---------------------------------------------------------------------------------
TOP = {d: float(torch.finfo(getattr(torch, d)).max) for d in ES}  # 3.39e38, 65504, 3.40e38


def assert_block_torch_cuda(q, s, x):
    """A block-scaled fp8 destination (q, s) against torch CUDA's quantisation of x: bytes (NaN bytes included) and
    scale_inv bits (any NaN equal to any NaN)."""
    want_q, want_s = block_fp8_oracle.torch_quantize(x.to(DEV))
    assert torch.equal(q.view(torch.uint8), want_q.view(torch.uint8))
    assert_same_bits_or_nan(s, want_s)


def assert_scaled_torch_cuda(q, s, x, g):
    """A channel- or tensor-scaled fp8 destination (q, s) against torch CUDA's quantisation of x, as
    assert_block_torch_cuda."""
    want_q, want_s = scaled_fp8_oracle.torch_quantize(x.to(DEV), g)
    assert torch.equal(q.view(torch.uint8), want_q.view(torch.uint8))
    assert_same_bits_or_nan(s, want_s)


# ---- groups of a destination window -----------------------------------------------------------------
def group_of(p: Pull, coord) -> tuple:
    """The destination group (block, row or matrix of the window) holding global element `coord`."""
    *lead, r, c = (x - o for x, o in zip(coord, p.dst[0]))
    if p.g == "block":
        return (*lead, r // BLOCK, c // BLOCK)
    return (*lead, r) if p.g == "channel" else tuple(lead)


def group_box(p: Pull, key) -> tuple:
    """Global index of every element of destination group `key`."""
    (*lo, r0, c0), (*_, n, k) = p.dst
    lead = tuple(o + i for o, i in zip(lo, key))
    if p.g == "block":
        br, bc = key[-2:]
        return lead + (slice(r0 + br * BLOCK, r0 + min(n, (br + 1) * BLOCK)), slice(c0 + bc * BLOCK, c0 + min(k, (bc + 1) * BLOCK)))
    if p.g == "channel":
        return lead + (slice(r0 + key[-1], r0 + key[-1] + 1), slice(c0, c0 + k))
    return lead + (slice(r0, r0 + n), slice(c0, c0 + k))


def n_groups(p: Pull) -> int:
    *lead, n, k = p.dst[1]
    m = int(np.prod(lead, dtype=np.int64))
    return m * -(-n // BLOCK) * -(-k // BLOCK) if p.g == "block" else m * n if p.g == "channel" else m


def fill_group(x, p: Pull, key, kind: str, seed: int):
    box = group_box(p, key)
    shape = tuple(x[box].shape)
    if kind == "zero":
        x[box] = torch.where(synth_f32(shape, seed) < 0, -0.0, 0.0)
    else:
        x[box] = synth_f32(shape, seed, spread=0) * torch.finfo(getattr(torch, p.dtype)).tiny * 0.5


KINDS = ("nan", "inf", "-inf", "zero", "subnormal")


def plant_special(x, p: Pull, coords, seed: int):
    """NaN, +Inf, -Inf, an all-zero (+-0) group and an all-subnormal group, each in its own destination group
    at the first spots that lie in one (one group of the window keeps finite data when it has several); -0 and
    single subnormals at the spots in the other groups."""
    x = x.float().clone()
    kinds = {}
    for j, c in enumerate(coords):
        key = group_of(p, c)
        if key not in kinds and len(kinds) < max(1, n_groups(p) - 1):
            kinds[key] = KINDS[len(kinds) % len(KINDS)]
            if kinds[key] in ("zero", "subnormal"):
                fill_group(x, p, key, kinds[key], seed + j)
        kind = kinds.get(key)
        if kind in ("nan", "inf", "-inf"):
            x[c] = float(kind)
        elif kind is None:
            x[c] = -0.0 if j % 2 else torch.finfo(getattr(torch, p.dtype)).tiny * 0.25
    return x.to(getattr(torch, p.dtype))


def near_top(x, p: Pull, coords, seed: int):
    """Values of magnitude [0.25, 1] x the largest finite value of the source dtype, +-that value at the spots."""
    top = TOP[p.dtype]
    u = synth_f32(tuple(x.shape), seed, spread=0)
    y = u.sign() * (0.25 + 0.75 * u.abs()) * top
    for j, c in enumerate(coords):
        y[c] = top if j % 2 == 0 else -top
    return y.to(getattr(torch, p.dtype))


def inputs(name: str, variant: str):
    from tests import test_quant_pull_regimes_cpu as qp_cpu  # the host suite imports this catalogue
    xs = qp_cpu.workload_inputs(name)
    if variant not in ("special", "near_top"):
        return xs
    w = WORKLOADS[name]
    tables, geom, *_ = qp_cpu.compiled(name)
    at = spots(tables, geom)
    plant = plant_special if variant == "special" else near_top
    return [plant(x, p, at.get(i, []), w.seed + 100 * i) for i, (p, x) in enumerate(zip(w.pulls, xs))]


# ---- one pull of several names ----------------------------------------------------------------------
class Pulled:
    """The names w0, w1, ... of `pulls` registered shard by shard (one source each), pulled into guarded
    destinations of `dst_dtype` (float8_e4m3fn or int8) and scales by one DirectWeightSyncDest with the scale format
    `scale_fmt`; `extra` handles and destinations join the pull."""

    def __init__(self, pulls, xs, extra_handles=None, extra_dests=None, scale_fmt=None, dst_dtype=E4M3):
        self.pulls, self.sources, self.shards, self.scale_fmt = tuple(pulls), [], {}, scale_fmt
        self.dst_dtype = dst_dtype
        self.handles, self.dests, self.scales, self.slices, self.bases = {}, {}, {}, {}, []
        try:
            for i, (p, x) in enumerate(zip(pulls, xs)):
                n = f"w{i}"
                self.handles[n], self.shards[n] = [], []
                for r, (off, loc) in enumerate(p.src):
                    shard = on_device(region(x, off, loc).contiguous(), p.shift(r))
                    src = DirectWeightSyncSource()
                    self.sources.append(src)
                    sl = TensorSlice(off, (r,), p.shape, loc, (len(p.src),))
                    self.handles[n].append(src.register({n: shard}, rank=r, tensor_slices={n: sl})[n])
                    self.shards[n].append(shard)
                qb, self.dests[n] = guarded(p.dst[1], dst_dtype)
                sb, self.scales[n] = guarded(dest_scale_shape(p.g, p.dst[1]), torch.float32)
                self.bases += [qb, sb]
                self.slices[n] = TensorSlice(p.dst[0], (0,), p.shape, p.dst[1], (1,))
        except BaseException:
            self.close()
            raise
        self.all_handles = {**self.handles, **(extra_handles or {})}
        self.all_dests = {**self.dests, **(extra_dests or {})}
        self.by_kw = {}
        for i, p in enumerate(self.pulls):
            self.by_kw.setdefault(KW[p.g], {})[f"w{i}"] = self.scales[f"w{i}"]
        self.sync = DirectWeightSyncDest()

    def pull(self):
        run(self.sync.pull(self.all_handles, self.all_dests, self.slices, **self.by_kw, scale_fmt=self.scale_fmt))

    def plan_dicts(self):
        """The (block, per-channel / per-tensor) plans of the destination format; the other format's stay empty."""
        fp8, int8 = (self.sync._block_plans, self.sync._scaled_plans), (self.sync._int8_block_plans, self.sync._int8_scaled_plans)
        mine, other = (int8, fp8) if self.dst_dtype == torch.int8 else (fp8, int8)
        assert not any(other), "plans of the other destination format"
        return mine

    def plans(self):
        return tuple(dict(p) for p in self.plan_dicts())

    def live_tables(self):
        """The tables of the plans the pull built, compiled on the host from the same windows and targets with
        the live device addresses; their size checked against plan_info."""
        tables, geom = compile_tables(self.pulls, self.sync._plan, self.handles, lambda b: b.window(0), self.dests, self.scales)
        want = plan_bytes(tables)
        for kind, plans in zip(("block", "scaled"), self.plan_dicts()):
            if kind in want:
                info = _native.plan_info(plans[0])
                assert (info.num_tiles, info.src_bytes) == want[kind], kind
            else:
                assert not plans, kind
        return tables, geom

    def check(self, xs):
        for i, (p, x) in enumerate(zip(self.pulls, xs)):
            n = f"w{i}"
            with named(f"w{i}: {p.describe()}"):
                assert_quantised(self.dests[n], self.scales[n], region(x, *p.dst), p.g, self.scale_fmt, self.dst_dtype)
        assert all(guards_intact(b) for b in self.bases)

    def update(self, xs):
        """New values in every source shard, in place; guard patterns over every destination and scale."""
        for i, (p, x) in enumerate(zip(self.pulls, xs)):
            for shard, (off, loc) in zip(self.shards[f"w{i}"], p.src):
                shard.copy_(region(x, off, loc).to(DEV))
            self.dests[f"w{i}"].view(torch.uint8).fill_(0xA5)
            self.scales[f"w{i}"].fill_(-3.0)

    def close(self):
        if hasattr(self, "sync"):
            self.sync.close()
        for src in self.sources:
            run(src.cleanup())


def assert_quantised(y, ys, x, g, scale_fmt=None, dst_dtype=E4M3):
    """The fp8 weight y and its scale_inv ys against the numpy oracle of the source region x (bit-exact in
    finite groups, NaN-agnostic in the others) and the torch CUDA composition (bit-exact, NaN bytes included),
    both in the scale format `scale_fmt`.  An int8 y: int8_source_oracle.assert_exact."""
    from tests import test_quant_pull_regimes_cpu as qp_cpu  # the host suite imports this catalogue
    if dst_dtype == torch.int8:
        int8_source_oracle.assert_exact(y, ys, x, g)
        return
    if scale_fmt is None:
        want_q, want_s = qp_cpu.oracle_quantize(x.float().numpy(), g)
    else:
        want_q, want_s = ue8m0_oracle.quantize(x.float().numpy(), g, scale_fmt=scale_fmt)
    q, s = y.view(torch.uint8).cpu().numpy(), ys.cpu().numpy()
    if g == "block":
        assert_block_fp8_equal(q, s, want_q, want_s)
    else:
        assert_scaled_fp8_equal(q, s, want_q, np.asarray(want_s, np.float32), g)
    if scale_fmt is not None:
        want_q, want_s = ue8m0_oracle.torch_quantize(x.to(DEV), g, scale_fmt=scale_fmt)
        want_s = want_s.reshape(ys.shape)
        assert torch.equal(y.view(torch.uint8), want_q.view(torch.uint8))  # NaN bytes included
        assert_same_bits_or_nan(ys, want_s)
        ue8m0_oracle.assert_pow2_over(ys, ue8m0_oracle.torch_quantize(x.to(DEV), g)[1])
    elif g == "block":
        assert_block_torch_cuda(y, ys, x)
    else:
        assert_scaled_torch_cuda(y, ys, x, g)


# ---- the regimes ------------------------------------------------------------------------------------
VARIANTS = ("finite", "special", "near_top", "update")


def run_regime(regime, variant, scale_fmt=None, dst_dtype=E4M3):
    """Pull the regime's workload in `variant` with the scale format `scale_fmt` into `dst_dtype` destinations,
    and check it (module doc)."""
    r = REGIMES[regime]
    w = WORKLOADS[r.workload]
    xs = inputs(r.workload, variant)
    where = f"{regime} ({r.doc}), {variant}, scale_fmt={scale_fmt}, {dst_dtype}: {w.describe()}"
    pulled = Pulled(w.pulls, xs, scale_fmt=scale_fmt, dst_dtype=dst_dtype)
    try:
        pulled.pull()
        tables, geom = pulled.live_tables()
        assert r.holds(tables, geom), f"not reached: {where}"
        with named(where):
            pulled.check(xs)
            if variant == "update":
                xs = [(rand_full(p.shape, getattr(torch, p.dtype), w.seed + 50 + i) * -0.5) for i, p in enumerate(w.pulls)]
                pulled.update(xs)
                before = pulled.plans()
                pulled.pull()
                assert pulled.plans() == before  # replayed, not rebuilt
                pulled.check(xs)
    finally:
        pulled.close()


# ---- random layouts with special values -------------------------------------------------------------
def boundary_spots(p: Pull, rng: random.Random, k: int = 8):
    """`k` global coordinates of the window drawn from the corners of every shard inside it, the rows and
    columns around block edges, and the ends and starts of consecutive rows."""
    (doff, dloc) = p.dst
    cands = []
    for off, loc in p.src:
        lo = [max(a, b) for a, b in zip(off, doff)]
        hi = [min(a + m, b + n) for a, m, b, n in zip(off, loc, doff, dloc)]
        if any(a >= b for a, b in zip(lo, hi)):
            continue
        lead = tuple(lo[:-2])
        for r in (lo[-2], hi[-2] - 1):
            for c in (lo[-1], hi[-1] - 1):
                cands.append(lead + (r, c))
    *lo, r0, c0 = doff
    *ln, n, kk = dloc
    for rr in (BLOCK - 1, BLOCK, rng.randrange(n)):
        for cc in (BLOCK - 1, BLOCK, 15, 16, kk - 1, 0):
            if rr < n and cc < kk:
                cands.append(tuple(o + rng.randrange(m) for o, m in zip(lo, ln)) + (r0 + rr, c0 + cc))
    return rng.sample(cands, min(k, len(cands)))


def plant_random(x, p: Pull, rng: random.Random, seed: int):
    """NaN, +-Inf, -0, a subnormal and the dtype's top at boundary spots; one group all zero, one subnormal."""
    x = x.float().clone()
    tiny = torch.finfo(getattr(torch, p.dtype)).tiny
    values = (float("nan"), float("inf"), float("-inf"), -0.0, tiny * 0.25, TOP[p.dtype])
    for j, c in enumerate(boundary_spots(p, rng)):
        x[c] = values[(j + seed) % len(values)]
    for j, kind in enumerate(("zero", "subnormal")):
        c = tuple(o + rng.randrange(m) for o, m in zip(*p.dst))
        fill_group(x, p, group_of(p, c), kind, seed + j)
    return x.to(getattr(torch, p.dtype))


def run_random_layout(seed, dst_dtype=E4M3):
    """Pull the layout drawn from `seed`, with special values, into a `dst_dtype` destination and check it."""
    rng = random.Random(19000 + seed)
    w = draw(rng, "quant", seed)
    p = Pull(("bfloat16", "float16", "float32")[seed % 3], w.shape, w.src, w.dst, w.out)
    x = plant_random(torch.randn(w.shape, generator=torch.Generator().manual_seed(seed)) * 0.05, p, rng, seed)
    pulled = Pulled((p,), [x], dst_dtype=dst_dtype)
    try:
        with named(f"seed {seed}: {p.describe()}"):
            pulled.pull()
            pulled.live_tables()
            pulled.check([x])
    finally:
        pulled.close()

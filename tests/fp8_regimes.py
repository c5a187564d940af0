"""Named branches of the requantising and dequantising kernels, decided from the compiled tables.

Every regime is a predicate over the record arrays ``_native.requant_fp8_compile_host`` (units, pieces,
tiles, n_groups) or ``_native.dequant_fp8_compile_host`` (tiles) return, plus the destination's geometry,
and names the workload that reaches it.  A workload is one pull: a global fp8 tensor cut into source
shards of one scale granularity, and one destination window.  The CPU suite compiles every workload on
host memory and replays it against the oracles; the H100 suites run it through ``DirectWeightSyncDest.pull``
(``run_regime``) and assert the regime again from the tables of the live plan's inputs.

Branches (csrc/requant_fp8.cu, csrc/dequant_fp8.cu):
  staged units      block targets (one group per 128x128 block) and per-channel bands of rows of at most
                    kSqStageBytes (32 KiB, kSqBandRows = 256 rows at most); pieces are ``vec`` (16-byte loads)
                    or byte-wise; the band's |x| fold is warp-reduced when a warp step stays in one row
                    (rows of >= 2048 bytes) and a per-lane atomicMax otherwise; a 16-element chunk that
                    straddles a source block or starts off a 16-byte column takes the per-element path.
  two-pass tiles    per-tensor targets and per-channel rows longer than the stage: tiles of at most
                    kSqTileElems (16384) elements, cut at 128 source columns for block sources; one amax word
                    per group; the tile at (row 0, column 0) of its group writes scale_inv.
  dequant tiles     at most 16384 elements and 256 rows (kDqTileRows: one staged scale per row), column tiles
                    for rows wider than 16384, ``vec`` when source and destination rows are 16-byte aligned.
"""

from __future__ import annotations

import random
from dataclasses import dataclass
from functools import partial
from typing import Callable

import numpy as np
import torch

from oracle import int8_source_oracle, ue8m0_oracle
from oracle.dequant_fp8_oracle import DST, GRANULARITIES, dequantize, torch_dequantize
from oracle.requant_fp8_oracle import SCALE_POISON, requantize, torch_requantize
from tests.helpers import (DEV, E4M3, assert_same_bits_or_nan, cleanup, guards_intact, named, pull_box, region,
                           register_boxes, shard_box)
from tests.test_dequant_fp8_cpu import local_scale as dq_local_scale
from tests.test_dequant_fp8_cpu import torch_bits
from tests.test_requant_fp8_cpu import CODE, fp8_full, global_scale, local_scale
from torchstore_b200 import _native
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, _add_dq_source
from torchstore_b200.planner import build_rects

STAGE_BYTES, TILE_ELEMS, BAND_ROWS, DQ_TILE_ROWS = 32768, 16384, 256, 256
ES = {"bfloat16": 2, "float16": 2, "float32": 4}
DTYPE_CODE = {"bfloat16": _native.TSB_BF16, "float16": _native.TSB_F16, "float32": _native.TSB_F32}


def split(shape, n, dim):
    """Even shards of ``shape`` along ``dim`` (the last shards may be short)."""
    return tuple(shard_box(shape, n, r, dim % len(shape)) for r in range(n))


def whole(shape):
    return ((0,) * len(shape), tuple(shape))


@dataclass(frozen=True)
class Workload:
    kind: str     # "requant" or "dequant"
    shape: tuple  # global shape [..., N, K] of the fp8 weight
    sg: str       # source scale granularity
    src: tuple    # source shards: ((offset, local shape), ...)
    dst: tuple    # destination window: (offset, local shape)
    out: str      # destination granularity (requant) or dtype (dequant)
    seed: int

    def describe(self) -> str:
        return f"{self.kind} {self.shape} {self.sg}-scaled src={list(self.src)} dst={self.dst} -> {self.out}"


@dataclass(frozen=True)
class Geometry:
    """What a predicate may know besides the tables: the destination window and the source shards."""
    dst: int       # address of the destination's element 0
    batch: int
    rows: int
    cols: int
    es: int        # destination element bytes
    sources: tuple  # (first byte, end) of every source shard

    def source_of(self, addr: int) -> int:
        return next(i for i, (lo, hi) in enumerate(self.sources) if lo <= addr < hi)

    def matrix_of(self, addr: int) -> int:
        return (addr - self.dst) // (self.rows * self.cols * self.es)

    def col_of(self, addr: int) -> int:
        return (addr - self.dst) % (self.cols * self.es) // self.es


def geometry(dst_ptr: int, dst_shape, es: int, sources, n_sources: int) -> Geometry:
    *lead, rows, cols = dst_shape
    spans = tuple((int(s.src), int(s.src) + int(s.batch * s.rows * s.cols)) for s in list(sources)[:n_sources])
    return Geometry(dst_ptr, int(np.prod(lead, dtype=np.int64)), rows, cols, es, spans)


# ---- workloads -----------------------------------------------------------------------------------
def _rq(shape, sg, src, dst, dg, seed):
    return Workload("requant", tuple(shape), sg, tuple(src), dst, dg, seed)


def _dq(shape, sg, src, dst, dtype, seed):
    return Workload("dequant", tuple(shape), sg, tuple(src), dst, dtype, seed)


WORKLOADS: dict[str, Workload] = {
    # block targets
    "rq_block_aligned": _rq((256, 384), "block", split((256, 384), 2, 0), whole((256, 384)), "block", 1),
    "rq_block_fsdp6_rows": _rq((300, 260), "block", split((300, 260), 6, 0), shard_box((300, 260), 2, 0, 0), "block", 2),
    "rq_block_tp_cols": _rq((256, 260), "block", (whole((256, 260)),), shard_box((256, 260), 2, 1, 1), "block", 3),
    "rq_block_col_shards": _rq((256, 260), "channel", split((256, 260), 2, 1), whole((256, 260)), "block", 4),
    "rq_block_moe": _rq((3, 130, 260), "block", split((3, 130, 260), 3, 1), whole((3, 130, 260)), "block", 5),
    # per-channel bands
    "rq_band_narrow": _rq((256, 512), "channel", split((256, 512), 2, 0), whole((256, 512)), "channel", 6),
    "rq_band_wide_moe": _rq((2, 64, 4096), "block", (whole((2, 64, 4096)),), whole((2, 64, 4096)), "channel", 7),
    "rq_band_ragged": _rq((300, 260), "block", split((300, 260), 6, 0), shard_box((300, 260), 2, 1, 0), "channel", 8),
    "rq_band_stage_bound": _rq((3, 32768), "block", (whole((3, 32768)),), whole((3, 32768)), "channel", 9),
    "rq_band_tall": _rq((600, 96), "channel", split((600, 96), 3, 0), whole((600, 96)), "channel", 10),
    "rq_band_col_shards": _rq((256, 260), "block", split((256, 260), 2, 1), whole((256, 260)), "channel", 11),
    # two-pass tiles
    "rq_tensor_aligned_moe": _rq((2, 256, 512), "tensor", split((2, 256, 512), 2, 0), whole((2, 256, 512)), "tensor", 12),
    "rq_tensor_ragged": _rq((300, 260), "channel", split((300, 260), 6, 0), shard_box((300, 260), 2, 0, 1), "tensor", 13),
    "rq_tensor_long_rows": _rq((4, 40000), "tensor", (whole((4, 40000)),), whole((4, 40000)), "tensor", 14),
    "rq_channel_long_block_src": _rq((3, 33000), "block", (whole((3, 33000)),), whole((3, 33000)), "channel", 15),
    "rq_channel_long_channel_src": _rq((3, 40000), "channel", split((3, 40000), 3, 0), whole((3, 40000)), "channel", 16),
    "rq_tensor_many_groups": _rq((260, 16, 64), "tensor", split((260, 16, 64), 2, 0), whole((260, 16, 64)), "tensor", 17),
    # dequant tiles
    **{f"dq_aligned_{d}": _dq((256, 512), "channel", split((256, 512), 2, 0), whole((256, 512)), d, 20 + i)
       for i, d in enumerate(ES)},
    **{f"dq_ragged_{d}": _dq((300, 260), "block", split((300, 260), 6, 0), shard_box((300, 260), 2, 0, 0), d, 23 + i)
       for i, d in enumerate(ES)},
    # source shards of 128 and 132 columns into 520-byte bf16 rows: the first is aligned, its destination is not
    "dq_misaligned_dst": _dq((64, 260), "tensor", (((0, 0), (64, 128)), ((0, 128), (64, 132))), whole((64, 260)),
                             "bfloat16", 26),
    "dq_wide_rows": _dq((3, 40008), "channel", (whole((3, 40008)),), whole((3, 40008)), "bfloat16", 27),
    "dq_narrow_rows": _dq((512, 48), "channel", split((512, 48), 2, 0), whole((512, 48)), "float32", 28),
}


# ---- predicates ----------------------------------------------------------------------------------
def _pieces(u, pieces):
    return pieces[int(u["piece0"]): int(u["piece0"]) + int(u["n_pieces"])]


def _units(tables, per_row):
    units, pieces, _, _ = tables
    return [(u, _pieces(u, pieces)) for u in units if int(u["per_row"]) == per_row]


def _block(f):
    return lambda tb, g: any(f(u, ps, g) for u, ps in _units(tb, 0))


def _band(f):
    return lambda tb, g: any(f(u, ps, g) for u, ps in _units(tb, 1))


def _tile(f):
    return lambda tb, g: any(f(t, tb[3], g) for t in tb[2])


def _straddles(p):
    """A 16-element chunk of the piece crosses a 128-column source block."""
    return bool(p["col_blocks"]) and any((int(p["col_phase"]) + c) % 128 > 112 for c in range(0, int(p["cols"]), 16))


def _dq_tile(f):
    return lambda tiles, g: any(f(t, g) for t in tiles)


@dataclass(frozen=True)
class Regime:
    workload: str
    holds: Callable  # (tables, Geometry) -> bool
    doc: str


REGIMES: dict[str, Regime] = {
    # requantise, staged block units
    "rq_block_unit_all_vec": Regime("rq_block_aligned", _block(lambda u, ps, g: (ps["vec"] == 1).all()),
                                    "block unit whose pieces all take 16-byte loads"),
    "rq_block_unit_byte_piece": Regime("rq_block_fsdp6_rows", _block(lambda u, ps, g: (ps["vec"] == 0).any()),
                                       "block unit with a byte-wise piece"),
    "rq_block_unit_straddling_chunk": Regime(
        "rq_block_tp_cols", _block(lambda u, ps, g: any(int(p["col_phase"]) % 16 and _straddles(p) for p in ps)),
        "block unit piece off the source's 16-column phase: chunks straddle a source block"),
    "rq_block_unit_piece_off_16_columns": Regime(
        "rq_block_col_shards", _block(lambda u, ps, g: (ps["col0"] % 16 != 0).any()),
        "block unit piece that starts off a 16-byte column of the unit"),
    "rq_block_unit_batch": Regime("rq_block_moe", _block(lambda u, ps, g: g.matrix_of(int(u["dst"])) > 0),
                                  "block unit of a matrix past the first of a stack"),
    # requantise, staged per-channel bands
    "rq_band_vec_short_rows": Regime(
        "rq_band_narrow", _band(lambda u, ps, g: int(u["cols"]) < 2048 and int(u["rows"]) > 1 and (ps["vec"] == 1).any()),
        "band of rows under 2048 B with a vec piece: warp steps span rows (per-lane atomicMax)"),
    "rq_band_vec_long_rows": Regime(
        "rq_band_wide_moe", _band(lambda u, ps, g: int(u["cols"]) >= 2048 and (ps["vec"] == 1).any()),
        "band of rows of >= 2048 B with a vec piece: warp steps inside one row (warp-reduced fold)"),
    "rq_band_byte_piece": Regime("rq_band_ragged", _band(lambda u, ps, g: (ps["vec"] == 0).any()),
                                 "band with a byte-wise piece"),
    "rq_band_one_row_at_stage_bound": Regime(
        "rq_band_stage_bound", _band(lambda u, ps, g: int(u["rows"]) == 1 and int(u["cols"]) == STAGE_BYTES),
        "band of one 32768-column row: the stage is exactly 32 KiB"),
    "rq_band_over_128_rows": Regime(
        "rq_band_tall", _band(lambda u, ps, g: int(u["rows"]) > 128 and int(u["cols"]) <= 128),
        "band of more than 128 rows of at most 128 columns"),
    "rq_band_several_sources": Regime(
        "rq_band_col_shards", _band(lambda u, ps, g: len({g.source_of(int(p["src"])) for p in ps}) > 1),
        "band assembled from pieces of several source shards"),
    "rq_band_source_scale_step": Regime(
        "rq_band_narrow", _band(lambda u, ps, g: ((ps["scale_step"] != 0) & (ps["rows"] > 1)).any()),
        "band piece with one source scale per row"),
    "rq_band_batch": Regime("rq_band_wide_moe", _band(lambda u, ps, g: g.matrix_of(int(u["dst"])) > 0),
                            "band of a matrix past the first of a stack"),
    # requantise, two-pass tiles
    "rq_tensor_tile_rows_vec": Regime("rq_tensor_aligned_moe", _tile(lambda t, n, g: t["rows"] > 1 and t["vec"] == 1),
                                      "per-tensor tile of several rows, 16-byte loads"),
    "rq_tensor_tile_rows_byte": Regime("rq_tensor_ragged", _tile(lambda t, n, g: t["rows"] > 1 and t["vec"] == 0),
                                       "per-tensor tile of several rows, byte loads"),
    "rq_tensor_tile_full_width": Regime(
        "rq_tensor_long_rows", lambda tb, g: tb[3] == g.batch and (tb[2]["cols"] == TILE_ELEMS).any()
        and (tb[2]["scale_inv"] != 0).sum() == tb[3],
        "per-tensor tiles of one 16384-column row segment, one scale_inv writer per group"),
    "rq_channel_long_rows_block_source": Regime(
        "rq_channel_long_block_src", lambda tb, g: g.cols > STAGE_BYTES and tb[3] == g.batch * g.rows
        and len(tb[2]) and (tb[2]["cols"] <= 128).all() and (tb[2]["scale_inv"] != 0).sum() == tb[3],
        "per-channel rows over 32 KiB from a block source: tiles cut at 128 source columns"),
    "rq_channel_long_rows_channel_source": Regime(
        "rq_channel_long_channel_src", lambda tb, g: g.cols > STAGE_BYTES and tb[3] == g.batch * g.rows
        and (tb[2]["cols"] == TILE_ELEMS).any() and (tb[2]["scale_inv"] != 0).sum() == tb[3],
        "per-channel rows over 32 KiB from a channel source: 16384-column tiles"),
    "rq_two_pass_source_scale_step": Regime(
        "rq_tensor_ragged", _tile(lambda t, n, g: t["scale_step"] != 0 and t["rows"] > 1),
        "two-pass tile with one source scale per row"),
    "rq_two_pass_over_256_groups": Regime("rq_tensor_many_groups", lambda tb, g: tb[3] > 256,
                                          "more than 256 amax words"),
    "rq_tile_batch": Regime("rq_tensor_aligned_moe", _tile(lambda t, n, g: g.matrix_of(int(t["dst"])) > 0),
                            "two-pass tile of a matrix past the first of a stack"),
    # dequantise
    **{f"dq_vec{v}_{d}": Regime(f"dq_{'aligned' if v else 'ragged'}_{d}",
                                _dq_tile(lambda t, g, v=v, d=d: t["vec"] == v and t["dst_dtype"] == DTYPE_CODE[d]),
                                f"{'16-byte' if v else 'byte-wise'} tile into {d}")
       for d in ES for v in (0, 1)},
    "dq_vec0_aligned_source": Regime(
        "dq_misaligned_dst", _dq_tile(lambda t, g: t["vec"] == 0 and t["src"] % 16 == 0 and t["rows"] > 1 and t["src_stride"] % 16 == 0),
        "byte-wise tile whose source rows are 16-byte aligned (the destination's are not)"),
    "dq_tile_full_width": Regime("dq_wide_rows", _dq_tile(lambda t, g: t["cols"] == TILE_ELEMS and t["rows"] == 1),
                                 "one-row tile of 16384 columns"),
    "dq_tile_column_remainder": Regime(
        "dq_wide_rows", _dq_tile(lambda t, g: t["cols"] < TILE_ELEMS and g.col_of(int(t["dst"])) > 0
                            and g.col_of(int(t["dst"])) % TILE_ELEMS == 0),
        "the last column tile of a row wider than 16384"),
    "dq_tile_256_rows_channel": Regime("dq_narrow_rows", _dq_tile(lambda t, g: t["rows"] == DQ_TILE_ROWS and t["scale_step"] == 4),
                                       "per-channel tile of 256 rows: every staged scale in use"),
    "dq_vec_tile_ragged_cols": Regime("dq_wide_rows", _dq_tile(lambda t, g: t["vec"] == 1 and t["cols"] % 16 != 0),
                                      "16-byte tile whose last chunk is partial"),
}


# ---- on the H100 ---------------------------------------------------------------------------------
def want_bits(q_full, full_scale, g, box, dtype):
    """The numpy oracle's bits of the `box` of `q_full` dequantised into `dtype`."""
    dst = str(dtype).replace("torch.", "")
    return dequantize(region(q_full, *box).view(torch.uint8).numpy(), dq_local_scale(full_scale, g, *box).numpy(), g,
                      box[0][-2], box[0][-1], dst)


def assert_dequant_oracle(y, want):
    """A dequantised destination y bit for bit the oracle's bits `want` wherever y is not NaN."""
    got = torch_bits(y.cpu())
    nan = torch.isnan(y.float()).cpu().numpy()
    assert np.array_equal(got[~nan], want[~nan])


def assert_dequant_torch_cuda(y, q_full, full_scale, g, box):
    """Bit-exact, NaN bytes included, against the torch CUDA rendering of the same region."""
    want = torch_dequantize(region(q_full, *box).to(DEV), dq_local_scale(full_scale, g, *box).to(DEV), g, box[0][-2],
                            box[0][-1], y.dtype)
    assert torch.equal(y.view(torch.uint8), want.view(torch.uint8))


def assert_requant_torch_cuda(q, s, q_full, full_scale, sg, box, dg, scale_fmt=None):
    """A requantised destination (q, s) bit-exact, NaN bytes included, against the torch CUDA composition of the
    same window."""
    args = (region(q_full, *box).to(DEV), local_scale(full_scale, sg, *box).to(DEV), sg, box[0][-2], box[0][-1], dg)
    want_q, want_s = ue8m0_oracle.torch_requantize(*args, scale_fmt=scale_fmt) if scale_fmt else torch_requantize(*args)
    if scale_fmt:
        ue8m0_oracle.assert_pow2_over(s, torch_requantize(*args)[1])
    assert torch.equal(q.view(torch.uint8), want_q.view(torch.uint8))
    assert_same_bits_or_nan(s.reshape(-1), want_s.reshape(-1))  # a NaN scale_inv's bits are torch's choice


def assert_requant_oracle(q, s, q_full, full_scale, sg, box, dg, scale_fmt=None):
    """A requantised destination (q, s) bit-exact against the numpy composition wherever it is not NaN."""
    args = (region(q_full, *box).view(torch.uint8).numpy(), local_scale(full_scale, sg, *box).numpy(), sg, box[0][-2],
            box[0][-1], dg)
    want_q, want_s = ue8m0_oracle.requantize(*args, scale_fmt=scale_fmt) if scale_fmt else requantize(*args)
    got_q = q.view(torch.uint8).cpu().numpy()
    nan = (want_q & 0x7F) == 0x7F
    assert np.array_equal(got_q[~nan], want_q[~nan])
    got_s, want_s = s.cpu().numpy().reshape(-1), np.asarray(want_s, np.float32).reshape(-1)
    ok = ~np.isnan(want_s)
    assert np.array_equal(got_s[ok].view(np.uint32), want_s[ok].view(np.uint32))


def live_tables(sync, dest, dest_scale=None, dg=None, int8_src=False):
    """Compile on the host the tables of the plan `sync` built for its one name: the same windows, sources and
    target it compiled from, with the live device addresses (`int8_src`: a dequantising plan of int8 handles, TSB_I8
    rects).  Checks their size against plan_info and returns (tables, Geometry)."""
    dev = dest.device.index
    pairs, sources = [], {}
    for op in sync._plan:
        pairs.append(DirectWeightSyncDest.op_windows(op, op.rdma_buffer.window(dev)))
        _add_dq_source(sources, op, dev)
    arr = _native.make_dq_source_array(max(1, len(sources)))
    for i, (_, s) in enumerate(sources.values()):
        arr[i] = s
    rects, n = build_rects(pairs, dequantise=int8_src)
    *lead, rows, cols = dest.shape
    if dg is None:
        tables = _native.dequant_fp8_compile_host(dev, rects, n, arr, len(sources))
        mine, other = (sync._int8_dequant_plans, sync._dequant_plans) if int8_src else (sync._dequant_plans, sync._int8_dequant_plans)
        assert not other, "dequantising plans of the other source format"
        info = _native.plan_info(mine[dev])
        count, read = len(tables), int((tables["rows"].astype(np.int64) * tables["cols"]).sum())
    else:
        for i in range(n):
            rects[i].src_dtype = rects[i].dst_dtype = _native.TSB_F8E4M3
        tgt = _native.make_sq_target_array(1)
        tgt[0] = _native.SqTarget(dest.data_ptr(), dest_scale.data_ptr(), dest.numel() // (rows * cols), rows, cols, CODE[dg], 0)
        tables = _native.requant_fp8_compile_host(dev, rects, n, arr, len(sources), tgt, 1)
        units, pieces, tiles, _ = tables
        info = _native.plan_info(sync._requant_plans[dev])
        count = len(units) + len(tiles)
        read = int((pieces["rows"].astype(np.int64) * pieces["cols"]).sum() + (tiles["rows"].astype(np.int64) * tiles["cols"]).sum())
    assert (info.num_tiles, info.src_bytes) == (count, read)
    return tables, geometry(dest.data_ptr(), tuple(dest.shape), dest.element_size(), arr, len(sources))


POISON = (float(SCALE_POISON[0]), float(SCALE_POISON[1]), 0.0, -0.5)  # Inf, NaN, 0, negative


def poison(s, seed):
    """Inf, NaN, 0 and -0.5 at four spread entries of a source scale (one of them if it has one entry)."""
    flat = s.reshape(-1)
    n = flat.numel()
    for k, i in enumerate(sorted({0, n // 3, 2 * n // 3, n - 1})):
        flat[i] = POISON[(k + seed) % len(POISON)]
    return s


def zero_first_group(q, w: Workload):
    """All-zero bytes over the first destination group of `w` (dequantising pulls: its first row)."""
    off, loc = w.dst
    *lead, n, k = loc
    h, kk = {"block": (min(128, n), min(128, k)), "channel": (1, k), "tensor": (n, k)}.get(w.out, (1, k))
    q.view(torch.uint8)[tuple(off[:-2]) + (slice(off[-2], off[-2] + h), slice(off[-1], off[-1] + kk))] = 0
    return q


def inputs(w: Workload, variant: str, src_dtype=E4M3):
    """The source weight (fp8 bytes, or int8 ones from int8_of) and its global scale of workload `w` in `variant`."""
    q = int8_source_oracle.int8_of(w.shape, w.seed) if src_dtype == torch.int8 else fp8_full(w.shape, w.seed)
    s = global_scale(w.sg, w.shape, w.seed)
    if variant == "poisoned_scale":
        s = poison(s, w.seed)
    elif variant == "zero_group":
        q = zero_first_group(q, w)
    return q, s


VARIANTS = ("finite", "poisoned_scale", "zero_group")


def run_regime(regime, variant, scale_fmt=None, src_dtype=E4M3):
    """Pull the regime's workload in `variant` (requantising ones with the scale format `scale_fmt`; dequantising
    ones from handles of `src_dtype`, float8_e4m3fn or int8) and check it."""
    r = REGIMES[regime]
    w = WORKLOADS[r.workload]
    int8 = src_dtype == torch.int8
    assert not (int8 and w.kind == "requant"), "int8 handles are not requantised"
    q, s = inputs(w, variant, src_dtype)
    sources, handles = register_boxes(q, list(w.src), granularity=w.sg, scale_of=partial(dq_local_scale, s, w.sg))
    where = f"{regime} ({r.doc}), {variant}, scale_fmt={scale_fmt}, {src_dtype}: {w.describe()}"
    if w.kind == "requant":
        sync, y, ys, bases = pull_box(handles, w.shape, w.dst, E4M3, granularity=w.out, requantize=True,
                                      scale_fmt=scale_fmt)
        tables, geom = live_tables(sync, y, ys, w.out)
        assert r.holds(tables, geom), f"not reached: {where}"
        with named(where):
            assert_requant_oracle(y, ys, q, s, w.sg, w.dst, w.out, scale_fmt)
            assert_requant_torch_cuda(y, ys, q, s, w.sg, w.dst, w.out, scale_fmt)
    else:
        sync, y, _, bases = pull_box(handles, w.shape, w.dst, DST[w.out])
        tables, geom = live_tables(sync, y, int8_src=int8)
        assert r.holds(tables, geom), f"not reached: {where}"
        with named(where):
            if int8:
                assert_int8_dequantised(y, q, s, w.sg, w.dst)
            else:
                assert_dequant_oracle(y, want_bits(q, s, w.sg, w.dst, DST[w.out]))
                assert_dequant_torch_cuda(y, q, s, w.sg, w.dst)
    assert all(guards_intact(b) for b in bases), where
    sync.close()
    cleanup(sources)


def assert_int8_dequantised(y, q, s, g, box):
    """A destination y dequantised from the `box` of int8 handles (q, global scale s): bit for bit the numpy oracle
    (NaN-agnostic) and the torch CUDA rendering (NaN bytes included)."""
    off, loc = box
    qr, sr = region(q, off, loc), local_scale(s, g, off, loc)
    assert_dequant_oracle(y, int8_source_oracle.dequantize(qr.numpy(), sr.numpy(), g, off[-2], off[-1], str(y.dtype)[6:]))
    want = int8_source_oracle.torch_dequantize(qr.to(DEV), sr.to(DEV), g, off[-2], off[-1], y.dtype)
    assert torch.equal(y.view(torch.uint8), want.view(torch.uint8))


WIDTHS = (16, 48, 64, 100, 128, 130, 260, 16384, 16400, 32768, 32784)
SRC_DTYPES = (torch.bfloat16, torch.float16, torch.float32)


def draw(rng: random.Random, kind: str, seed: int) -> Workload:
    """One random pull of `kind` ("quant", "dequant" or "requant")."""
    k = rng.choice(WIDTHS)
    n = rng.randint(1, max(1, min(400, 300_000 // k)))
    shape = (rng.randint(2, 4), n, k) if rng.random() < 0.3 else (n, k)
    layout = rng.choice(["rows", "cols", "replica"] + (["ep"] * (len(shape) == 3)))
    if layout == "rows":
        src = split(shape, rng.randint(2, 6), -2)
    elif layout == "cols":
        src = split(shape, rng.randint(2, 4), -1)
    elif layout == "replica":
        src = split(shape, 2, -2) * 2
    else:
        src = split(shape, shape[0], 0)
    src = tuple(b for b in src if 0 not in b[1])
    tp = rng.choice(["whole", "rows", "cols"])
    dst = whole(shape) if tp == "whole" else shard_box(shape, 2, rng.randint(0, 1), len(shape) - (2 if tp == "rows" else 1))
    if 0 in dst[1]:
        dst = whole(shape)
    sg = rng.choice(SRC_DTYPES) if kind == "quant" else rng.choice(GRANULARITIES)
    out = rng.choice(list(DST)) if kind == "dequant" else rng.choice(GRANULARITIES)
    return Workload(kind, shape, str(sg).replace("torch.", ""), src, dst, out, seed)

"""Named branches of source-side quantisation (csrc/source_quant.cu and the two-pass tiles it borrows from
csrc/scaled_fp8.cu), decided from the compiled tables.

Every regime is a predicate over the record arrays ``_native.source_quant_compile_host`` returns (units, tiles,
n_groups), plus the targets they were compiled from, and names the workload that reaches it.  A workload is
one ``register(quantize=...)`` call: a list of targets, each a bf16/f16/f32 shard with its shape (leading dims
make a stack), granularity, global offset (row0, col0) and a misalignment of its source address in elements.
The CPU suite compiles every workload on host memory and replays it against the oracle; the H100 suite
registers it (``run_regime``) and asserts the regime again from the tables of the live addresses.

Branches:
  units             blocks (one group: the part of a global 128x128 block inside the shard) and per-channel bands
                    of at most min(256, 32768 / row pitch, 1024 / chunks per row) rows, one CTA each and one launch
                    per source dtype (bf16, f16, f32, in that order in the table); ``vec`` units take 16-byte
                    loads, the others load element by element.  In a band the |x| fold of a warp step is
                    warp-reduced when its 32 chunks sit in one row (chunks per row a multiple of 32) and a per-lane
                    atomicMax otherwise; rows of 33 or more chunks that are no multiple of 32 mix both.
  two-pass tiles    per-tensor matrices and per-channel rows over 32 KiB: tiles of at most 16384 contiguous
                    elements, one amax word per group, the group's first tile writes scale_inv; ``vec`` when the
                    tile's source is 16-byte aligned and its bytes a multiple of 16.
"""

from __future__ import annotations

from dataclasses import dataclass
from typing import Callable

import numpy as np
import torch

from oracle import int8_source_oracle, ue8m0_oracle
from oracle.source_quant_oracle import bits_of, element_scales, quantize, synth_f32, torch_quantize, widen
from tests.helpers import DEV, E4M3, guarded, guards_intact, named, run
from tests.test_source_quant_cpu import CODE as GCODE
from tests.test_source_quant_cpu import compile_host
from torchstore_b200 import _native
from torchstore_b200.direct_weight_sync import DirectWeightSyncSource, source_scale_shapes
from torchstore_b200.launch import Plans
from torchstore_b200.transport.types import TensorSlice

STAGE_BYTES, TILE_ELEMS, BAND_ROWS, UNIT_CHUNKS = 32768, 16384, 256, 1024
ES = {"bfloat16": 2, "float16": 2, "float32": 4}
CODE = {"bfloat16": _native.TSB_BF16, "float16": _native.TSB_F16, "float32": _native.TSB_F32}
NAME = {v: k for k, v in CODE.items()}


@dataclass(frozen=True)
class Target:
    dtype: str        # "bfloat16", "float16" or "float32"
    shape: tuple      # local shape [..., N, K]
    granularity: str  # "block", "channel" or "tensor"
    row0: int = 0     # global offset of the shard in its last two dims
    col0: int = 0
    misalign: int = 0  # source address this many elements past a 16-byte boundary

    def describe(self) -> str:
        mis = f" +{self.misalign}" if self.misalign else ""
        return f"{self.granularity} {self.dtype}{list(self.shape)} at ({self.row0}, {self.col0}){mis}"


@dataclass(frozen=True)
class Workload:
    targets: tuple  # of Target, one name each in one register()
    seed: int

    def describe(self) -> str:
        return "; ".join(t.describe() for t in self.targets)


def _w(seed, *targets):
    return Workload(tuple(targets), seed)


WORKLOADS: dict[str, Workload] = {
    # block units, 16-byte and element-wise loads per dtype
    **{f"block_aligned_{d}": _w(100 + i, Target(d, (256, 384), "block")) for i, d in enumerate(ES)},
    **{f"block_misaligned_{d}": _w(110 + i, Target(d, (129, 257), "block", 37, 70, 1)) for i, d in enumerate(ES)},
    # partial first and last block rows and columns: rows 91/128/81, columns 58/128/14
    "block_mid_block": _w(120, Target("bfloat16", (300, 200), "block", 37, 70)),
    # per-channel bands
    "channel_rows_of_6_chunks": _w(130, Target("float16", (600, 96), "channel", 37, 0)),
    "channel_rows_of_64_chunks": _w(131, Target("bfloat16", (64, 1024), "channel")),
    "channel_rows_of_33_chunks": _w(132, Target("float32", (70, 520), "channel", 5, 70)),
    "channel_tall_bf16": _w(133, Target("bfloat16", (600, 64), "channel", 100, 0)),
    "channel_tall_f32": _w(134, Target("float32", (520, 16), "channel")),
    "channel_rows_of_32_chunks": _w(135, Target("bfloat16", (100, 512), "channel")),
    "channel_stack_bands": _w(136, Target("float16", (3, 100, 64), "channel", 28, 0)),
    "channel_misaligned": _w(137, Target("bfloat16", (50, 300), "channel", 0, 0, 3)),
    # one row of exactly 32 KiB, and the first widths past it (two-pass)
    **{f"channel_stage_bound_{d}": _w(140 + i, Target(d, (3, STAGE_BYTES // ES[d]), "channel")) for i, d in enumerate(ES)},
    "channel_past_stage_bf16": _w(143, Target("bfloat16", (3, STAGE_BYTES // 2 + 1), "channel")),
    "channel_past_stage_f32": _w(144, Target("float32", (2, STAGE_BYTES // 4 + 1), "channel")),
    # two-pass tiles
    "tensor_remainder_stack": _w(150, Target("float16", (3, 130, 260), "tensor", 100, 5)),
    "tensor_many_matrices": _w(151, Target("bfloat16", (300, 16, 64), "tensor")),
    "channel_long_many_rows": _w(152, Target("bfloat16", (260, STAGE_BYTES // 2 + 1), "channel")),
    **{f"tensor_misaligned_{d}": _w(153 + i, Target(d, (130, 260), "tensor", 0, 0, 1)) for i, d in enumerate(ES)},
    # several targets in one plan
    "three_dtypes": _w(160, Target("float32", (130, 200), "block", 0, 70), Target("bfloat16", (200, 130), "channel", 64, 0),
                       Target("float16", (140, 260), "block", 37, 0), Target("bfloat16", (2, 64, 300), "block")),
    "units_and_tiles": _w(161, Target("bfloat16", (300, 260), "block", 37, 70), Target("float32", (2, 130, 260), "tensor"),
                          Target("float16", (40, 1000), "channel")),
}


# ---- predicates ----------------------------------------------------------------------------------
def _units(tables, per_row):
    units = tables[0]
    return [u for u in units if int(u["per_row"]) == per_row]


def chunks(u) -> int:
    return (int(u["cols"]) + 15) // 16


def _block(f):
    return lambda tb, tg: any(f(u) for u in _units(tb, 0))


def _band(f):
    return lambda tb, tg: any(f(u) for u in _units(tb, 1))


def _tile(f):
    return lambda tb, tg: any(f(t) for t in tb[1])


def target_of(targets, addr: int):
    """The target whose source holds byte `addr`, and its element size."""
    for t in targets:
        es = ES[NAME[int(t.src_dtype)]]
        if t.src <= addr < t.src + t.batch * t.rows * t.cols * es:
            return t, es
    raise AssertionError(f"no target holds address {addr:#x}")


def crosses_matrix(u, targets) -> bool:
    """A band whose rows run over the end of one matrix of a stack into the next."""
    t, es = target_of(targets, int(u["src"]))
    first = (int(u["src"]) - t.src) // (t.cols * es)
    return first // t.rows != (first + int(u["rows"]) - 1) // t.rows


def first_last_partial(units) -> bool:
    """Partial block rows and columns at both ends of the shard: two distinct row and column counts under 128."""
    rows = {int(u["rows"]) for u in units if int(u["rows"]) < 128}
    cols = {int(u["cols"]) for u in units if int(u["cols"]) < 128}
    return len(rows) >= 2 and len(cols) >= 2 and (units["rows"] == 128).any() and (units["cols"] == 128).any()


def one_writer_per_group(tiles, n_groups) -> bool:
    return len(tiles) > 0 and (tiles["scale_inv"] != 0).sum() == n_groups and \
        len({int(t["group"]) for t in tiles if int(t["scale_inv"])}) == n_groups


def dtype_runs(units) -> list:
    """The source dtypes of the units in table order, one entry per run (one launch each)."""
    order = [NAME[int(d)] for d in units["src_dtype"]]
    return [d for i, d in enumerate(order) if i == 0 or order[i - 1] != d]


@dataclass(frozen=True)
class Regime:
    workload: str
    holds: Callable  # (tables, targets) -> bool
    doc: str


REGIMES: dict[str, Regime] = {
    # block units
    **{f"block_unit_vec_{d}": Regime(f"block_aligned_{d}",
                                     _block(lambda u, d=d: int(u["vec"]) == 1 and NAME[int(u["src_dtype"])] == d
                                            and int(u["rows"]) * chunks(u) == UNIT_CHUNKS),
                                     f"{d} block unit of 128x128 (1024 chunks) with 16-byte loads")
       for d in ES},
    **{f"block_unit_bytewise_{d}": Regime(f"block_misaligned_{d}",
                                          _block(lambda u, d=d: int(u["vec"]) == 0 and NAME[int(u["src_dtype"])] == d),
                                          f"{d} block unit loaded element by element")
       for d in ES},
    "block_partial_first_and_last": Regime("block_mid_block", lambda tb, tg: first_last_partial(tb[0]),
                                           "partial first and last block rows and columns of a shard at a mid-block offset"),
    # per-channel bands
    "band_lane_atomics": Regime("channel_rows_of_6_chunks", _band(lambda u: int(u["rows"]) > 1 and chunks(u) < 32),
                                "band of rows under 32 chunks: every warp step spans rows (per-lane atomicMax)"),
    "band_warp_reduced": Regime("channel_rows_of_64_chunks", _band(lambda u: chunks(u) % 32 == 0 and int(u["rows"]) > 1),
                                "band of rows of a multiple of 32 chunks: every warp step in one row (warp-reduced)"),
    "band_mixed_fold": Regime("channel_rows_of_33_chunks", _band(lambda u: chunks(u) > 32 and chunks(u) % 32 != 0
                                                                 and int(u["rows"]) > 1),
                              "band of 520-column rows: warp steps inside one row and across two"),
    "band_256_rows": Regime("channel_tall_bf16", _band(lambda u: int(u["rows"]) == BAND_ROWS),
                            "bf16 band of 256 rows: amax and scale slots past 128"),
    "band_256_rows_f32": Regime("channel_tall_f32", _band(lambda u: int(u["rows"]) == BAND_ROWS and NAME[int(u["src_dtype"])] == "float32"),
                                "f32 band of 256 rows of one chunk"),
    "band_1024_chunks": Regime("channel_rows_of_32_chunks", _band(lambda u: int(u["rows"]) > 1 and int(u["rows"]) * chunks(u) == UNIT_CHUNKS),
                               "band of 32 rows of 32 chunks: all 1024 chunk slots of the CTA in use"),
    "band_crosses_matrix": Regime("channel_stack_bands", lambda tb, tg: any(crosses_matrix(u, tg) for u in _units(tb, 1)),
                                  "band whose rows run from one matrix of a stack into the next"),
    "band_bytewise": Regime("channel_misaligned", _band(lambda u: int(u["vec"]) == 0 and int(u["rows"]) > 1),
                            "band loaded element by element"),
    **{f"band_one_row_at_stage_bound_{d}": Regime(
        f"channel_stage_bound_{d}",
        _band(lambda u, d=d: int(u["rows"]) == 1 and int(u["cols"]) * ES[d] == STAGE_BYTES and NAME[int(u["src_dtype"])] == d),
        f"{d} band of one row of exactly 32 KiB")
       for d in ES},
    "two_pass_first_width_past_stage_bf16": Regime(
        "channel_past_stage_bf16", lambda tb, tg: len(tb[0]) == 0 and tb[2] == 3 and (tb[1]["cols"] == TILE_ELEMS).any()
        and (tb[1]["cols"] == 1).any() and one_writer_per_group(tb[1], tb[2]),
        "bf16 rows of 16385 columns: two-pass, a 16384-column tile and a 1-column remainder per row"),
    "two_pass_first_width_past_stage_f32": Regime(
        "channel_past_stage_f32", lambda tb, tg: len(tb[0]) == 0 and tb[2] == 2 and (tb[1]["cols"] == STAGE_BYTES // 4 + 1).all(),
        "f32 rows of 8193 columns: two-pass, one tile per row"),
    # two-pass tiles
    "tensor_tiles_with_remainder": Regime(
        "tensor_remainder_stack", lambda tb, tg: tb[2] == 3 and (tb[1]["cols"] == TILE_ELEMS).any()
        and ((tb[1]["cols"] % TILE_ELEMS) != 0).any() and one_writer_per_group(tb[1], tb[2]),
        "per-tensor tiles of a stack, 16384-element tiles and a remainder, one scale_inv writer per group"),
    "two_pass_over_256_groups_tensor": Regime("tensor_many_matrices", lambda tb, tg: tb[2] > 256 and one_writer_per_group(tb[1], tb[2]),
                                              "per-tensor stack of 300 matrices: more than 256 amax words"),
    "two_pass_over_256_groups_channel": Regime(
        "channel_long_many_rows", lambda tb, tg: tb[2] > 256 and len(tb[0]) == 0 and one_writer_per_group(tb[1], tb[2]),
        "260 per-channel rows over 32 KiB: more than 256 amax words"),
    **{f"two_pass_bytewise_{d}": Regime(f"tensor_misaligned_{d}",
                                        _tile(lambda t, d=d: int(t["vec"]) == 0 and NAME[int(t["src_dtype"])] == d),
                                        f"{d} two-pass tile loaded element by element")
       for d in ES},
    # several targets in one plan
    "three_dtype_launches": Regime("three_dtypes", lambda tb, tg: dtype_runs(tb[0]) == ["bfloat16", "float16", "float32"],
                                   "units of all three source dtypes: three launches that advance through one table"),
    "units_and_tiles": Regime("units_and_tiles", lambda tb, tg: len(tb[0]) > 0 and len(tb[1]) > 0 and len(set(tb[0]["per_row"].tolist())) == 2,
                              "block and band units beside two-pass tiles in one plan"),
}


def plan_bytes(tables) -> tuple[int, int]:
    """(work items, source bytes read) of compiled tables: what plan_info reports as num_tiles and src_bytes."""
    units, tiles, _ = tables
    es = lambda a: np.array([ES[NAME[int(d)]] for d in a["src_dtype"]], dtype=np.int64)  # noqa: E731
    read = int((units["rows"].astype(np.int64) * units["cols"] * es(units)).sum()) if len(units) else 0
    read += int((tiles["cols"].astype(np.int64) * es(tiles)).sum()) if len(tiles) else 0
    return len(units) + len(tiles), read


# ---- on the H100 ---------------------------------------------------------------------------------
def assert_exact(q: torch.Tensor, s: torch.Tensor, x: torch.Tensor, g: str, r0: int, c0: int, scale_fmt=None):
    """Bit-exact against torch CUDA everywhere (NaN bytes included) and against the numpy oracle on finite groups,
    both in the scale format `scale_fmt`."""
    tq, tsc = ue8m0_oracle.torch_quantize(x.to(q.device), g, r0, c0, scale_fmt=scale_fmt)
    assert torch.equal(q.view(torch.uint8), tq.view(torch.uint8))
    assert torch.equal(s.view(torch.int32), tsc.reshape(s.shape).view(torch.int32))
    xf = widen(bits_of(x.cpu()), str(x.dtype)[6:])
    want_q, want_s = ue8m0_oracle.quantize(xf, g, r0, c0, scale_fmt=scale_fmt) if scale_fmt else quantize(xf, g, r0, c0)
    want_s = np.asarray(want_s, np.float32).reshape(tuple(s.shape))
    if scale_fmt:
        ue8m0_oracle.assert_pow2_over(s, torch_quantize(x.to(q.device), g, r0, c0)[1])
    got_q, got_s = q.view(torch.uint8).cpu().numpy(), s.cpu().numpy()
    fin = np.isfinite(element_scales(want_s, g, want_q.shape, r0, c0))
    assert np.array_equal(got_q[fin], want_q[fin])
    fs = np.isfinite(want_s)
    assert np.array_equal(got_s[fs].view(np.uint32), want_s[fs].view(np.uint32))


def on_device(x: torch.Tensor, misalign: int = 0) -> torch.Tensor:
    """`x` on the GPU, starting `misalign` elements into a fresh allocation (not 16-byte aligned if > 0) with
    4096 elements of slack after it, so that reads past a shard's end stay inside the allocation."""
    flat = torch.zeros(x.numel() + 4096, dtype=x.dtype, device=DEV)
    out = flat[misalign: misalign + x.numel()].view(x.shape)
    out.copy_(x.to(DEV))
    return out


def local_slice(shape, row0, col0, global_shape=None, rank=0, ranks=1):
    lead = tuple(shape[:-2])
    gshape = global_shape or lead + (row0 + shape[-2], col0 + shape[-1])
    offsets = (0,) * len(lead) + (row0, col0)
    return TensorSlice(offsets, (rank,), tuple(gshape), tuple(shape), (ranks,))


# ---- the regimes ------------------------------------------------------------------------------------
def group_boxes(t: Target):
    """Index tuples of the first and the last group of a target's shard."""
    *lead, n, k = t.shape
    first_m, last_m = (0,) * len(lead), tuple(e - 1 for e in lead)
    if t.granularity == "block":
        r1, c1 = min(n, 128 - t.row0 % 128), min(k, 128 - t.col0 % 128)
        lr, lc = max(0, (t.row0 + n - 1) // 128 * 128 - t.row0), max(0, (t.col0 + k - 1) // 128 * 128 - t.col0)
        return first_m + (slice(0, r1), slice(0, c1)), last_m + (slice(lr, n), slice(lc, k))
    if t.granularity == "channel":
        return first_m + (slice(0, 1), slice(None)), last_m + (slice(n - 1, n), slice(None))
    return first_m + (slice(None), slice(None)), last_m + (slice(None), slice(None))


def plant(x: torch.Tensor, t: Target, kind: str, seed: int) -> torch.Tensor:
    """Special values in the first and the last group of `x` (in its dtype): +Inf and -Inf, or NaN, at the
    first element of the first group and the last element of the last; or both groups all zero or subnormal."""
    x = x.float().clone()
    first, last = group_boxes(t)
    first_elem, last_elem = (0,) * len(t.shape), tuple(e - 1 for e in t.shape)
    if kind in ("inf", "nan"):
        x[first_elem] = float("inf") if kind == "inf" else float("nan")
        x[last_elem] = float("-inf") if kind == "inf" else float("nan")
    elif kind == "zero":
        x[first] = 0
        x[last] = 0
    elif kind == "subnormal":
        tiny = torch.finfo(getattr(torch, t.dtype)).tiny
        for box in (first, last):
            x[box] = synth_f32(tuple(x[box].shape), seed, spread=0) * tiny * 0.5
    return x.to(getattr(torch, t.dtype))


def register_workload(name, xs, scale_fmt=None, quant_dtype=None):
    """One register() of every target of workload `name` (values `xs`), in the scale format `scale_fmt` and the
    staging dtype `quant_dtype` -> (source, handles, device shards)."""
    w = WORKLOADS[name]
    src = DirectWeightSyncSource()
    sd, slices, quant = {}, {}, {}
    for i, (t, x) in enumerate(zip(w.targets, xs)):
        sd[f"t{i}"] = on_device(x, t.misalign)
        slices[f"t{i}"] = local_slice(t.shape, t.row0, t.col0)
        quant[f"t{i}"] = t.granularity
    handles = src.register(sd, rank=0, tensor_slices=slices, quantize=quant, scale_fmt=scale_fmt, quant_dtype=quant_dtype)
    return src, handles, sd


def live_tables(src, handles, w, quant_dtype=None):
    """Compile on the host the targets register() built, from the staging it allocated and the handles'
    offsets (for int8 staging with TSB_I8); check their size against plan_info -> (tables, targets)."""
    targets = []
    for i, t in enumerate(w.targets):
        fp8, scale, local = src._quantized[f"t{i}"]
        buf = handles[f"t{i}"].rdma_buffer
        rows, cols = local.shape[-2:]
        targets.append(_native.SourceQuantTarget(local.data_ptr(), fp8.data_ptr(), scale.data_ptr(), local.numel() // (rows * cols),
                                                 rows, cols, buf.row0, buf.col0, CODE[t.dtype], GCODE[t.granularity]))
    if quant_dtype == torch.int8:
        arr = _native.make_source_quant_target_array(len(targets))
        for i, t in enumerate(targets):
            arr[i] = t
        tables = _native.source_quant_compile_host(0, arr, len(targets), dst_dtype=_native.TSB_I8)
    else:
        tables = compile_host(targets)
    info = _native.plan_info(src._quant_plans[0])
    assert (info.num_tiles, info.src_bytes) == plan_bytes(tables)
    return tables, targets


def check_staging(src, w, xs, scale_fmt=None, quant_dtype=None):
    for i, (t, x) in enumerate(zip(w.targets, xs)):
        q, s, _ = src._quantized[f"t{i}"]
        with named(t.describe()):
            if quant_dtype == torch.int8:
                int8_source_oracle.assert_exact(q, s, x, t.granularity, t.row0, t.col0)
            else:
                assert_exact(q, s, x, t.granularity, t.row0, t.col0, scale_fmt)


VARIANTS = ("finite", "inf", "nan", "zero", "subnormal", "refresh")


def run_regime(regime, variant, scale_fmt=None, quant_dtype=None):
    """Register the regime's workload in `variant` with the scale format `scale_fmt` and the staging dtype
    `quant_dtype`, and check it (module doc)."""
    from tests import test_source_quant_regimes_cpu as sq_cpu  # the host suite imports this catalogue
    r = REGIMES[regime]
    w = WORKLOADS[r.workload]
    xs = sq_cpu.workload_inputs(r.workload)
    if variant not in ("finite", "refresh"):
        xs = [plant(x, t, variant, w.seed + i) for i, (t, x) in enumerate(zip(w.targets, xs))]
    src, handles, sd = register_workload(r.workload, xs, scale_fmt, quant_dtype)
    where = f"{regime} ({r.doc}), {variant}, scale_fmt={scale_fmt}, quant_dtype={quant_dtype}: {w.describe()}"
    try:
        tables, targets = live_tables(src, handles, w, quant_dtype)
        assert r.holds(tables, targets), f"not reached: {where}"
        with named(where):
            check_staging(src, w, xs, scale_fmt, quant_dtype)
            if variant == "refresh":
                xs = [synth_f32(t.shape, w.seed + 50 + i).to(x.dtype) * 0.25 for i, (t, x) in enumerate(zip(w.targets, xs))]
                for i, x in enumerate(xs):
                    sd[f"t{i}"].copy_(x.to(DEV))
                assert src.refresh() == len(w.targets)
                check_staging(src, w, xs, scale_fmt, quant_dtype)
    finally:
        run(src.cleanup())


def run_guarded(name, scale_fmt=None, quant_dtype=None):
    from tests import test_source_quant_regimes_cpu as sq_cpu  # the host suite imports this catalogue
    w = WORKLOADS[name]
    xs = sq_cpu.workload_inputs(name)
    targets, outs = [], []
    for t, x in zip(w.targets, xs):
        sv = on_device(x, t.misalign)
        sshape = source_scale_shapes(t.granularity, t.shape, t.row0, t.col0)[0]
        qbase, q = guarded(t.shape, quant_dtype or E4M3)
        sbase, s = guarded(sshape, torch.float32)
        rows, cols = t.shape[-2:]
        targets.append(_native.SourceQuantTarget(sv.data_ptr(), q.data_ptr(), s.data_ptr(), x.numel() // (rows * cols), rows, cols,
                                                 t.row0, t.col0, CODE[t.dtype], GCODE[t.granularity]))
        outs.append((sv, q, s, qbase, sbase))
    plans = Plans.build_source_quant({0: targets}, _native.TSB_QUANT_UE8M0 if scale_fmt else 0,
                                     _native.TSB_I8 if quant_dtype == torch.int8 else _native.TSB_F8E4M3)
    try:
        for _ in range(2):
            plans.launch()
            plans.synchronize()
    finally:
        plans.close()
    for t, x, (_, q, s, qbase, sbase) in zip(w.targets, xs, outs):
        with named(f"{name}: {t.describe()}"):
            if quant_dtype == torch.int8:
                int8_source_oracle.assert_exact(q, s, x, t.granularity, t.row0, t.col0)
            else:
                assert_exact(q, s, x, t.granularity, t.row0, t.col0, scale_fmt)
            assert guards_intact(qbase) and guards_intact(sbase)

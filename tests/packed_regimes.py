"""Named regimes of packed destinations (``pull(..., packed=...)``), their numpy reference and their host compile.

A regime is a geometry: one packed destination cut into parts, and for each part's source a global shape and a
handle layout (row, column and 2-D mesh shards, uneven shards, replicated handles).  A route gives the geometry its
dtypes: byte copies and fused casts of bf16/f16/f32 handles, quantising into fp8 (float32 and UE8M0 scales) and
int8, dequantising scaled fp8 and int8 handles, requantising and verbatim pulls.  ``spec(regime, route)`` is one
``DirectWeightSyncDest.pull``; the ``mixed_routes*`` regimes are pulls of several names on different routes.

The reference (:func:`expect`) shares no code with the package: every source is rendered as a global array by the
existing numpy oracles (a scaled handle dequantised with its own scale and ``(row0, col0)``, an element-wise
source converted by the fp8 oracle), ``oracle/packed_oracle.fill`` applies the parts, and grouped routes quantise
the filled array with the quantisers' oracles.

:func:`host_pull` plans a spec on host memory through ``DirectWeightSyncDest._build_plan`` and the package's
route verdicts, compiles it with the host compilers exactly as ``DirectWeightSyncDest._compile`` splits the work,
and replays the tables with the oracle interpreters.  The H100 suite pulls the same specs on the device.
"""

from __future__ import annotations

import itertools
import random
from dataclasses import dataclass, field

import numpy as np
import torch

import workloads
from oracle import (block_fp8_oracle, dequant_fp8_oracle, fp8_oracle, int8_oracle, int8_source_oracle, packed_oracle,
                    requant_fp8_oracle, scaled_fp8_oracle, ue8m0_oracle)
from torchstore_b200 import _native
from torchstore_b200.direct_weight_sync import (DirectWeightSyncDest, PackedPart, RDMAWeightHandle, _add_dq_source,
                                                _as_grid, _is_int8, _lift, _quant_target, _route_handles, scale_grid,
                                                scale_fmt_flags, source_scale_shapes)
from torchstore_b200.planner import StridedMem, build_rects
from torchstore_b200.transport.types import TensorSlice

from tests import helpers
from tests.helpers import cuda_like, rect_fields, region

BLOCK = 128
E4M3, E5M2 = torch.float8_e4m3fn, torch.float8_e5m2
DT = {"bfloat16": torch.bfloat16, "float16": torch.float16, "float32": torch.float32, "e4m3": E4M3, "e5m2": E5M2,
      "int8": torch.int8}
SCALED = ("e4m3", "int8")  # what a scaled handle holds
CODE = {"float16": 4, "bfloat16": 5, "float32": 6, "e4m3": 8, "e5m2": 9}  # the ABI's TSB_* dtype codes
BITS = {1: torch.uint8, 2: torch.int16, 4: torch.int32}
SENTINEL = 0x5A  # every byte of a destination before the pull
SCALE_SENTINEL = -1.0
VARIANTS = ("finite", "special", "update")


# ---- specs -----------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Src:
    """A source tensor: global shape, what its handles hold, their scale granularity (scaled handles) and
    their boxes ((global offsets, local shape), one per handle; a box listed twice is a replica)."""
    shape: tuple
    dtype: str
    g: str | None
    boxes: tuple


@dataclass(frozen=True)
class Dst:
    """A destination: local shape, dtype, scale granularity (scaled destinations) and its parts, or for an
    unpacked name the global offsets of its window in the source of the same name."""
    shape: tuple
    dtype: str
    g: str | None = None
    parts: tuple | None = None
    window: tuple | None = None


@dataclass(frozen=True)
class Spec:
    sources: dict
    dests: dict
    requantize: bool = False
    verbatim: bool = False
    scale_fmt: str | None = None

    def kw(self) -> dict:
        return dict(requantize=self.requantize, verbatim=self.verbatim, scale_fmt=self.scale_fmt)

    def packed(self) -> dict:
        return {n: d.parts for n, d in self.dests.items() if d.parts is not None}

    def route_of(self, name: str) -> str:
        """The route this spec means for ``name``, decided from the spec alone: copy, cast, quant, dequant,
        requant or verbatim."""
        d = self.dests[name]
        srcs = {p.source for p in d.parts} if d.parts is not None else {name}
        scaled = {self.sources[s].g is not None for s in srcs}
        assert len(scaled) == 1, name
        if d.g is None:
            if scaled == {True}:
                return "dequant"
            return "copy" if {self.sources[s].dtype for s in srcs} == {d.dtype} else "cast"
        if scaled == {False}:
            return "quant"
        return "verbatim" if self.verbatim else "requant"


@dataclass(frozen=True)
class Route:
    """The dtypes a geometry is pulled with."""
    kind: str          # copy, cast, quant, dequant, requant or verbatim
    src: str           # what the handles hold
    out: str           # the destination's dtype
    g: str | None = None    # the destination's scale granularity
    sg: str | None = None   # the handles' scale granularity
    fmt: str | None = None  # scale_fmt


def _routes() -> dict[str, Route]:
    out = {"copy_bf16": Route("copy", "bfloat16", "bfloat16"), "copy_f32": Route("copy", "float32", "float32")}
    for s, d in (("bfloat16", "float32"), ("float32", "bfloat16"), ("float16", "float32"), ("float32", "float16"),
                 ("bfloat16", "e4m3"), ("float16", "e5m2"), ("float32", "e4m3"), ("bfloat16", "e5m2")):
        out[f"cast_{s}_{d}"] = Route("cast", s, d)
    for g, s in (("block", "bfloat16"), ("channel", "float16"), ("tensor", "float32"), ("block", "float32")):
        out[f"quant_fp8_{g}_{s}"] = Route("quant", s, "e4m3", g)
    for g, s in (("block", "bfloat16"), ("channel", "float32"), ("tensor", "float16")):
        out[f"quant_ue8m0_{g}_{s}"] = Route("quant", s, "e4m3", g, fmt="ue8m0")
    for g, s in (("block", "float16"), ("channel", "bfloat16"), ("tensor", "float32")):
        out[f"quant_int8_{g}_{s}"] = Route("quant", s, "int8", g)
    for q in SCALED:
        for sg, o in (("block", "bfloat16"), ("channel", "float32"), ("tensor", "float16")):
            out[f"dq_{q}_{sg}_{o}"] = Route("dequant", q, o, sg=sg)
    for sg, g in (("block", "block"), ("block", "channel"), ("channel", "block"), ("tensor", "tensor"), ("tensor", "block")):
        out[f"rq_{sg}_{g}"] = Route("requant", "e4m3", "e4m3", g, sg)
    out["rq_block_block_ue8m0"] = Route("requant", "e4m3", "e4m3", "block", "block", "ue8m0")
    for q in SCALED:
        for g in ("block", "channel", "tensor"):
            out[f"vb_{q}_{g}"] = Route("verbatim", q, q, g, g)
    return out


ROUTES = _routes()
ELEMENT = [r for r, v in ROUTES.items() if v.kind in ("copy", "cast")]
QUANT = [r for r, v in ROUTES.items() if v.kind == "quant"]
DEQUANT = [r for r, v in ROUTES.items() if v.kind == "dequant"]
REQUANT = [r for r, v in ROUTES.items() if v.kind == "requant"]
ALL_BUT_VERBATIM = ELEMENT + QUANT + DEQUANT + REQUANT


# ---- handle layouts ---------------------------------------------------------------------------------------------
def whole(shape) -> tuple:
    return (((0,) * len(shape), tuple(shape)),)


def shard(shape, dim: int, n: int) -> tuple:
    """torch.chunk-style Shard(dim) over n ranks (uneven when n does not divide the dim); empty shards dropped."""
    out = [workloads.shard_box(shape, n, r, ("S", dim)) for r in range(n)]
    return tuple((o, l) for o, l in out if 0 not in l)


def cuts(shape, dim: int, bounds) -> tuple:
    edges = [0, *bounds, shape[dim]]
    out = []
    for a, b in zip(edges, edges[1:]):
        off, loc = [0] * len(shape), list(shape)
        off[dim], loc[dim] = a, b - a
        out.append((tuple(off), tuple(loc)))
    return tuple(out)


def mesh(shape, da: int, ba, db: int, bb) -> tuple:
    """A 2-D mesh: the intersections of cuts along dims da and db."""
    out = []
    for (oa, la), (ob, lb) in itertools.product(cuts(shape, da, ba), cuts(shape, db, bb)):
        off, loc = list(oa), list(la)
        off[db], loc[db] = ob[db], lb[db]
        out.append((tuple(off), tuple(loc)))
    return tuple(out)


def replicated(shape, dim: int, n: int) -> tuple:
    """(Replicate, Shard(dim)) over 2 x n ranks: every shard twice."""
    return shard(shape, dim, n) * 2


# ---- the catalogue ------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Regime:
    """A geometry: the packed destination ``w`` and its sources ``{name: (shape, boxes)}``, the routes it is pulled
    on, and a predicate over the host run of ``branch_route`` showing it reaches the branch it is named for."""
    shape: tuple
    parts: tuple
    sources: dict
    routes: tuple
    branch_route: str
    holds: object  # (HostRun) -> bool
    doc: str
    custom: object = None  # (route) -> Spec, for the regimes of several names


def P(source, index, offsets) -> PackedPart:
    return PackedPart(source, tuple(index), tuple(offsets))


def S(a, b):
    return slice(a, b)


def spec(regime: str, route: str) -> Spec:
    r, ro = REGIMES[regime], ROUTES.get(route)
    if r.custom is not None:
        return r.custom(route)
    srcs = {n: Src(shape, ro.src, ro.sg, boxes) for n, (shape, boxes) in r.sources.items()}
    return Spec(srcs, {"w": Dst(r.shape, ro.out, ro.g, r.parts)}, requantize=ro.kind == "requant",
                verbatim=ro.kind == "verbatim", scale_fmt=ro.fmt)


# predicates -----------------------------------------------------------------------------------------------------
def _pieces(tables):
    units, pieces = tables[0], tables[1]
    return [(u, pieces[int(u["piece0"]): int(u["piece0"]) + int(u["n_pieces"])]) for u in units]


def _block_from_three_parts(run) -> bool:
    return any(len({run.owner(int(p["src"]))[0] for p in ps}) >= 3 for _, ps in _pieces(run.tables["block"]))


def _vec_and_scalar_pieces(run) -> bool:
    ps = run.tables["block"][1]
    return bool((ps["vec"] == 1).any() and (ps["vec"] == 0).any())


def _source_phase_differs(run) -> bool:
    """A requant piece whose source block row (global, in the source) is not its destination block row."""
    units, pieces = run.tables["requant"][0], run.tables["requant"][1]
    for u, ps in _pieces((units, pieces)):
        d_row = run.dest_row(int(u["dst"]))
        for p in ps:
            name, h, (r, _) = run.owner(int(p["src"]))
            if (r // BLOCK) != (d_row + int(p["row0"])) // BLOCK:
                return True
    return False


def _two_tensor_scales(run) -> bool:
    tiles = run.tables["dequant"]
    return bool((tiles["scale_step"] == 0).all() and len(set(tiles["scale"].tolist())) >= 2)


def _stride0_unit_dims(k: int):
    def holds(run) -> bool:
        ws = run.windows["w"]
        return len(ws) > 0 and all(len(op.dest_dropped) == k and all(
            src.shape[d] == 1 and src.stride[d] == 0 for d in op.dest_dropped) for op, (src, _) in zip(run.ops, ws))
    return holds


def _dedup_and_mesh_edges(run) -> bool:
    """c's four handles (two replicas of two shards) give two ops, b's part meets all four tiles of its mesh."""
    n_c = sum(1 for op in run.ops if run.owner_of_buffer(op.rdma_buffer) == "c")
    n_b = sum(1 for op in run.ops if run.owner_of_buffer(op.rdma_buffer) == "b")
    return n_c == 2 and len(run.spec.sources["c"].boxes) == 4 and n_b == 4


def _rect_reads(run) -> dict:
    """{source name: global rows of the first byte of each compiled copy rect reading it}."""
    out = {}
    for addr in rect_fields(run.tables["copy"][0])["src"]:
        name, _, (row, _) = run.owner(int(addr))
        out.setdefault(name, set()).add(row)
    return out


def _kv_twin(run) -> bool:
    """The compiled copy rects of TP8 rank 3 read k and v only inside kv head 3 // (8 / n_kv) = 1, the head rank 2 reads
    too: kv heads replicated beyond the kv head count."""
    cfg = workloads.QWEN3_MOE
    hd, head = cfg["head_dim"] // 16, 3 // (8 // cfg["n_kv_heads"])
    reads = _rect_reads(run)
    kv = [p.source for p in run.spec.dests["w"].parts[1:]]
    return len(kv) == 2 and all(reads[n] and min(reads[n]) == head * hd and max(reads[n]) < (head + 1) * hd for n in kv)


def _has_holes(run) -> bool:
    """The compiled copy plan, replayed from sources full of a marker byte into a sentinel destination, writes exactly
    the parts' boxes: the elements outside every part (there are some) are written by no rect."""
    covered = np.zeros(run.spec.dests["w"].shape, dtype=bool)
    for p in run.spec.dests["w"].parts:
        covered[p.dest_index] = True
    dest = run.dests["w"]
    for hs in run.handles.values():
        for h in hs:
            h.rdma_buffer.shard.view(torch.uint8).fill_(0xA5)
    dest.view(torch.uint8).fill_(SENTINEL)
    table, tiles, info = run.tables["copy"]
    fp8_oracle.replay_plan(table, tiles, info.tile_bytes // 16, nan_mode=1)
    written = (dest.contiguous().view(torch.uint8).reshape(dest.shape + (-1,)) != SENTINEL).all(-1).numpy()
    return not covered.all() and np.array_equal(written, covered)


def _straddling_block(run) -> bool:
    return any(len({run.owner(int(p["src"]))[0] for p in ps}) == 2 for _, ps in _pieces(run.tables["requant"]))


def _every_route_compiled(run) -> bool:
    return {"copy", "block", "scaled", "dequant"} <= set(run.tables) and ("requant" in run.tables or "verbatim" in run.tables)


QWEN_HF = workloads.qwen3_moe_layout(workloads.QWEN3_MOE, n_layers=1, scale=16, n_experts=2, with_embeddings=False)
QKV = "model.layers.0.self_attn.qkv_proj.weight"


def _kv_regime():
    shape, parts, _ = workloads.vllm_tp_layout(QWEN_HF, workloads.QWEN3_MOE, 8, 3)[QKV]
    srcs = {p.source: (QWEN_HF[p.source][0], shard(QWEN_HF[p.source][0], 0, 3)) for p in parts}
    return tuple(shape), tuple(parts), srcs


def _mixed(route: str) -> Spec:
    """One pull of several names: copy, cast, quantising (block, channel, tensor, int8), dequantising (fp8 and int8)
    and requantising packed names next to an unpacked one (``mixed``), or UE8M0 quantising and verbatim names
    (``ue8m0_verbatim``)."""
    def rows(shape, n):
        return shard(shape, 0, n)
    srcs = {
        "q": Src((64, 136), "bfloat16", None, rows((64, 136), 2)),
        "k": Src((40, 136), "bfloat16", None, rows((40, 136), 3)),
        "v": Src((40, 136), "bfloat16", None, whole((40, 136))),
        "fa": Src((100, 150), "float32", None, rows((100, 150), 2)),
        "fb": Src((60, 150), "float32", None, whole((60, 150))),
        "sa": Src((256, 200), "e4m3", "block", rows((256, 200), 2)),
        "sb": Src((384, 200), "e4m3", "block", cuts((384, 200), 0, (128, 256))),
        "ia": Src((90, 140), "int8", "channel", rows((90, 140), 3)),
        "ib": Src((50, 140), "int8", "channel", whole((50, 140))),
        "u": Src((100, 64), "bfloat16", None, rows((100, 64), 3)),
    }
    qkv = (P("q", (S(0, 64), S(0, 136)), (0, 0)), P("k", (S(64, 90), S(0, 136)), (7, 0)),
           P("v", (S(90, 120), S(0, 136)), (10, 0)))
    cast = (P("fa", (S(0, 70), S(0, 150)), (13, 0)), P("fb", (S(70, 130), S(0, 150)), (0, 0)))
    dq = (P("sa", (S(0, 100), S(0, 200)), (30, 0)), P("sb", (S(100, 256), S(0, 200)), (200, 0)))
    aligned = (P("sa", (S(0, 128), S(0, 200)), (128, 0)), P("sb", (S(128, 384), S(0, 200)), (0, 0)))
    dqi = (P("ia", (S(0, 33), S(0, 140)), (41, 0)), P("ib", (S(33, 83), S(0, 140)), (0, 0)))
    if route == "mixed":
        dests = {"copy": Dst((120, 136), "bfloat16", parts=qkv), "cast": Dst((130, 150), "bfloat16", parts=cast),
                 "qb": Dst((120, 136), "e4m3", "block", qkv), "qc": Dst((120, 136), "e4m3", "channel", qkv),
                 "qt": Dst((120, 136), "e4m3", "tensor", qkv), "qi": Dst((120, 136), "int8", "block", qkv),
                 "dq": Dst((256, 200), "bfloat16", parts=dq), "dqi": Dst((83, 140), "float32", parts=dqi),
                 "rq": Dst((256, 200), "e4m3", "channel", dq), "u": Dst((60, 64), "bfloat16", window=(30, 0))}
        return Spec(srcs, dests, requantize=True)
    dests = {"copy": Dst((120, 136), "bfloat16", parts=qkv), "qb": Dst((120, 136), "e4m3", "block", qkv),
             "qc": Dst((130, 150), "e4m3", "channel", cast), "dq": Dst((256, 200), "float16", parts=dq),
             "vb": Dst((384, 200), "e4m3", "block", aligned), "u": Dst((100, 64), "bfloat16", window=(0, 0))}
    return Spec(srcs, dests, verbatim=True, scale_fmt="ue8m0")


def _catalogue() -> dict[str, Regime]:
    kv_shape, kv_parts, kv_srcs = _kv_regime()
    col_starts = (0, 3, 16, 100, 128, 200, 300)
    col_src_offsets = ((0, 0), (5, 1), (10, 16), (1, 7), (0, 128), (9, 33))
    # source rows of whole 16-byte units in bf16/f16 (16-byte strides), so the aligned parts take 16-byte loads
    col_src_widths = [-(-(b - a + o[1] + 9) // 8) * 8 for a, b, o in zip(col_starts, col_starts[1:], col_src_offsets)]
    drop_lead_parts = tuple(P(f"e{e}{j}", (e, j, S(0, 96), S(0, 160)), (128 * ((e + j) % 2), 0))
                            for e in range(2) for j in range(2))
    return {
        "row_parts_unaligned": Regime(
            (242, 200),
            (P("a", (S(0, 1), S(0, 200)), (37, 3)), P("b", (S(1, 16), S(0, 200)), (250, 0)),
             P("c", (S(16, 112), S(0, 200)), (96, 40)), P("d", (S(112, 242), S(0, 200)), (0, 0))),
            {"a": ((40, 210), shard((40, 210), 0, 2)), "b": ((300, 200), shard((300, 200), 0, 3)),
             "c": ((256, 256), cuts((256, 256), 0, (128,))), "d": ((130, 200), whole((130, 200)))},
            tuple(ALL_BUT_VERBATIM + ["vb_e4m3_channel", "vb_int8_channel"]), "quant_fp8_block_bfloat16",
            _block_from_three_parts, "parts of 1, 15, 96 and 130 rows: a block gathered from three parts"),
        "col_parts": Regime(
            (160, 300),
            tuple(P(f"s{i}", (S(0, 160), S(a, b)), o) for i, (a, b, o) in
                  enumerate(zip(col_starts, col_starts[1:], col_src_offsets))),
            {f"s{i}": ((170, w), shard((170, w), 0, 2)) for i, w in enumerate(col_src_widths)},
            tuple(ALL_BUT_VERBATIM), "quant_fp8_block_bfloat16", _vec_and_scalar_pieces,
            "parts side by side at columns 0, 3, 16, 100, 128, 200: 16-byte and element-wise pieces in one plan"),
        "src_phase": Regime(
            (256, 256),
            (P("a", (S(0, 160), S(0, 256)), (101, 37)), P("b", (S(160, 256), S(0, 256)), (3, 130))),
            {"a": ((420, 300), cuts((420, 300), 0, (100, 230))), "b": ((300, 400), cuts((300, 400), 1, (170,)))},
            tuple(ALL_BUT_VERBATIM), "rq_block_block", _source_phase_differs,
            "sources read from rows 101 and 3, columns 37 and 130, of shards at rows 100 / 230 and column 170"),
        "per_tensor_sources": Regime(
            (192, 256),
            (P("a", (S(0, 128), S(0, 256)), (0, 0)), P("b", (S(128, 192), S(0, 256)), (0, 0))),
            {"a": ((128, 256), whole((128, 256))), "b": ((64, 256), whole((64, 256)))},
            tuple(ELEMENT[:2] + ["quant_fp8_tensor_float32", "dq_e4m3_tensor_float16", "dq_int8_tensor_float16",
                                 "rq_tensor_tensor", "rq_tensor_block"]),
            "dq_e4m3_tensor_float16", _two_tensor_scales, "one destination group fed by two per-tensor sources"),
        "drop_row_dim": Regime(
            (64, 3, 200), tuple(P(f"s{k}", (S(0, 64), k, S(0, 200)), (3 * k, k)) for k in range(3)),
            {f"s{k}": ((80, 210), shard((80, 210), 0, 2)) for k in range(3)},
            tuple(ALL_BUT_VERBATIM), "copy_bf16", _stride0_unit_dims(1), "dest[R, 3, C] filled at [:, k, :]"),
        "drop_col_dim": Regime(
            (100, 64, 2), tuple(P(f"s{k}", (S(0, 100), S(0, 64), k), (5 * k, 3)) for k in range(2)),
            {f"s{k}": ((110, 70), shard((110, 70), 1, 2)) for k in range(2)},
            tuple(ELEMENT + QUANT), "copy_bf16", _stride0_unit_dims(1),
            "dest[R, C, 2] filled at [..., k] (dequantising and requantising pulls refuse it: "
            "test_scaled_sources_into_a_dropped_column_dim_are_refused)"),
        "drop_two_lead": Regime(
            (2, 2, 96, 160), drop_lead_parts,
            {f"e{e}{j}": ((256, 160), shard((256, 160), 0, 2)) for e in range(2) for j in range(2)},
            tuple(ALL_BUT_VERBATIM + [f"vb_{q}_{g}" for q in SCALED for g in ("block", "channel", "tensor")]),
            "copy_bf16", _stride0_unit_dims(2), "dest[E, 2, I, H] with ints on dims 0 and 1 from 2-D sources"),
        "sharded_sources": Regime(
            (200, 300),
            (P("a", (S(0, 130), S(0, 300)), (7, 5)), P("b", (S(130, 200), S(0, 150)), (33, 21)),
             P("c", (S(130, 200), S(150, 300)), (0, 0))),
            {"a": ((260, 310), shard((260, 310), 1, 3)), "b": ((140, 200), mesh((140, 200), 0, (70,), 1, (100,))),
             "c": ((70, 150), replicated((70, 150), 0, 2))},
            tuple(ALL_BUT_VERBATIM), "copy_bf16", _dedup_and_mesh_edges,
            "Shard(1) uneven, a 2-D mesh cut at 37 rows / 79 columns into its part, and replicated handles read once"),
        "kv_replicated": Regime(
            kv_shape, kv_parts, kv_srcs, tuple(ELEMENT[:3] + QUANT + DEQUANT + REQUANT), "copy_bf16", _kv_twin,
            "Qwen3-MoE qkv_proj at TP8 rank 3 (4 kv heads): k and v replicated across ranks 2 and 3"),
        "holes": Regime(
            (64, 200), (P("a", (S(0, 20), S(0, 150)), (5, 3)), P("b", (S(30, 64), S(10, 200)), (0, 0))),
            {"a": ((30, 160), shard((30, 160), 0, 2)), "b": ((40, 190), whole((40, 190)))},
            tuple(ELEMENT + DEQUANT), "copy_bf16", _has_holes, "elements outside every part are left alone"),
        "w13_straddle": Regime(
            (1, 192, 256), (P("gate", (0, S(0, 96), S(0, 256)), (96, 0)), P("up", (0, S(96, 192), S(0, 256)), (96, 0))),
            {"gate": ((768, 256), whole((768, 256))), "up": ((768, 256), whole((768, 256)))},
            ("quant_fp8_block_bfloat16", "dq_e4m3_block_bfloat16", "rq_block_block", "rq_block_channel",
             "rq_block_block_ue8m0"),
            "rq_block_block", _straddling_block,
            "Qwen3-30B-A3B w13 at TP8: 96-row gate and up halves, block row 0 straddles both"),
        "mixed_routes": Regime((), (), {}, ("mixed",), "mixed", _every_route_compiled,
                               "copy, cast, quantise, dequantise and requantise names in one pull", custom=_mixed),
        "mixed_routes_ue8m0_verbatim": Regime((), (), {}, ("ue8m0_verbatim",), "ue8m0_verbatim",
                                              lambda run: {"copy", "block", "scaled", "dequant", "verbatim"} <= set(run.tables),
                                              "UE8M0 quantising, verbatim, dequantising and copy names in one pull",
                                              custom=_mixed),
    }


REGIMES = _catalogue()
CASES = [(r, ro) for r, reg in REGIMES.items() for ro in reg.routes]


# ---- data ----------------------------------------------------------------------------------------------------------
@dataclass
class Data:
    """The global value of every source (CPU, in what its handles hold) and each handle's own scale."""
    full: dict
    scales: dict = field(default_factory=dict)  # name -> [local scale per handle]


def _scale_field(src: Src, gen) -> torch.Tensor:
    """Block and channel: a global scale anchored at the origin; tensor: one base per matrix of the lead dims."""
    shape = dequant_fp8_oracle.scale_shape(src.g, src.shape)
    return torch.rand(shape, generator=gen) * (0.02 if src.dtype == "int8" else 0.004) + 1e-4


def local_scale(src: Src, fld: torch.Tensor, k: int) -> torch.Tensor:
    """Handle k's scale: the groups its shard touches (block, channel), or its matrices' base times a factor of its
    box (tensor: shards of one tensor carry scales of their own; replicas agree)."""
    off, loc = src.boxes[k]
    *lead_off, r0, c0 = off
    *lead, n, c = loc
    li = tuple(slice(o, o + e) for o, e in zip(lead_off, lead))
    if src.g == "block":
        return fld[li + (slice(r0 // BLOCK, -(-(r0 + n) // BLOCK)), slice(c0 // BLOCK, -(-(c0 + c) // BLOCK)))].contiguous()
    if src.g == "channel":
        return fld[li + (slice(r0, r0 + n),)].contiguous()
    distinct = list(dict.fromkeys(src.boxes))
    return (fld[li] * (1 + 0.375 * distinct.index(src.boxes[k]))).contiguous()


def make_data(spec: Spec, seed: int, special: bool = False) -> Data:
    gen = torch.Generator().manual_seed(seed)
    data = Data({})
    for name, src in spec.sources.items():
        if src.dtype == "int8":
            x = torch.randint(-128, 128, src.shape, generator=gen, dtype=torch.int8)
        else:
            x = torch.randn(src.shape, generator=gen) * torch.exp2(torch.randint(-4, 5, src.shape[:-1] + (1,), generator=gen))
            x = x.to(DT[src.dtype]) if src.dtype != "e4m3" else (x * 8).to(E4M3)
        data.full[name] = x
        if src.g is not None:
            data.scales[name] = _scale_field(src, gen)
    if special:
        plant_specials(spec, data)
    for name, src in spec.sources.items():
        if src.g is not None:
            fld = data.scales[name]
            data.scales[name] = [local_scale(src, fld, k) for k in range(len(src.boxes))]
    return data


SPECIAL_FLOATS = (float("nan"), float("inf"), float("-inf"), "subnormal", 0.0, "-subnormal", "max")


def spots(spec: Spec) -> list[tuple[str, tuple]]:
    """(source, global index) of each part's box corners and of the elements its box holds at destination rows and
    columns 127 / 128 (group edges), in part order."""
    out = []
    for d in spec.dests.values():
        for p in d.parts or (PackedPart("", (), ()),):
            if not p.source:
                continue
            box = [(e, e + 1) if isinstance(e, int) else (e.start, e.stop) for e in p.dest_index]
            kept = [k for k, e in enumerate(p.dest_index) if not isinstance(e, int)]
            (r0, r1), (c0, c1) = box[-2], box[-1]
            cand = [(r0, c0), (r1 - 1, c1 - 1), (r0, c1 - 1), (r1 - 1, c0)]
            cand += [(r, c) for r in (127, 128) for c in (c0, 127, 128) if r0 <= r < r1 and c0 <= c < c1]
            for r, c in dict.fromkeys(cand):
                idx = [s for s, _ in box]
                idx[-2], idx[-1] = r, c
                src_idx = tuple(o + idx[k] - box[k][0] for o, k in zip(p.source_offsets, kept))
                out.append((p.source, src_idx))
    return out


def plant_specials(spec: Spec, data: Data) -> None:
    """NaN, +-Inf, subnormals, zeros and the largest finite value at every spot of the unscaled sources; NaN bytes
    (fp8) and Inf, NaN, zero, subnormal-product and negative scales at the spots of scaled ones; and the source rows
    of the first part's first destination row all zero (a zero channel, a block with a zero row)."""
    for i, (name, idx) in enumerate(spots(spec)):
        src, x = spec.sources[name], data.full[name]
        if src.g is None:
            v = SPECIAL_FLOATS[i % len(SPECIAL_FLOATS)]
            if isinstance(v, str):
                fi = torch.finfo(x.dtype)
                v = {"subnormal": fi.smallest_normal / 4, "-subnormal": -fi.smallest_normal / 2, "max": fi.max}[v]
            x[idx] = v
            continue
        if src.dtype == "e4m3" and i % 3 == 0:
            x.view(torch.uint8)[idx] = 0x7F if i % 2 else 0xFF
        fld = data.scales[name]
        g_idx = tuple(idx[:-2]) + ((idx[-2] // BLOCK, idx[-1] // BLOCK) if src.g == "block" else
                                   (idx[-2], 0) if src.g == "channel" else ())
        fld[g_idx] = (float("inf"), float("nan"), 0.0, 2.0 ** -140, -0.5)[i % 5]
    for d in spec.dests.values():
        if d.parts:
            p = d.parts[0]
            row = [s for s, e in enumerate(p.dest_index) if not isinstance(e, int)]
            lo = list(p.source_offsets)
            hi = [o + (e.stop - e.start) for o, e in zip(lo, (p.dest_index[k] for k in row))]
            hi[-2] = lo[-2] + 1
            data.full[p.source][tuple(slice(a, b) for a, b in zip(lo, hi))] = 0
            break


# ---- the reference --------------------------------------------------------------------------------------------------
def _bits(t: torch.Tensor) -> np.ndarray:
    return t.contiguous().view(BITS[t.element_size()]).numpy()


def _from_bits(a: np.ndarray, dtype: str) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a)).view(DT[dtype])


def convert(x: torch.Tensor, src: str, out: str) -> torch.Tensor:
    """``x`` (in ``src``) in ``out`` by the fp8 oracle's conversion (torch's ``.to()`` semantics)."""
    if src == out:
        return x.clone()
    y = torch.empty(x.shape, dtype=DT[out])
    xc = x.contiguous()
    fp8_oracle.convert(xc.data_ptr(), CODE[src], y.data_ptr(), CODE[out], xc.numel(), nan_mode=1)
    return y


def dequantised(src: Src, data: Data, name: str, out: str) -> torch.Tensor:
    """The global array a dequantising pull of ``name``'s handles writes in ``out``: each handle dequantised with its
    own scale and (row0, col0)."""
    g = torch.zeros(src.shape, dtype=DT[out])
    full = data.full[name]
    for (off, loc), scale in zip(src.boxes, data.scales[name]):
        q = full[tuple(slice(o, o + e) for o, e in zip(off, loc))]
        if src.dtype == "e4m3":
            bits = dequant_fp8_oracle.dequantize(q.contiguous().view(torch.uint8).numpy(), scale.numpy(), src.g,
                                                 off[-2], off[-1], out)
        else:
            with np.errstate(all="ignore"):
                y = (q.numpy().astype(np.float32) *
                     dequant_fp8_oracle.expand(scale.numpy(), tuple(loc), src.g, off[-2], off[-1])).astype(np.float32)
            bits = dequant_fp8_oracle.narrow(y, out)
        g[tuple(slice(o, o + e) for o, e in zip(off, loc))] = _from_bits(bits, out)
    return g


def scale_of_element(src: Src, data: Data, name: str) -> np.ndarray:
    """float32 [source shape]: the scale of the handle and group each element is read from (first handle wins)."""
    out = np.zeros(src.shape, dtype=np.float32)
    done = np.zeros(src.shape, dtype=bool)
    for (off, loc), scale in zip(src.boxes, data.scales[name]):
        box = tuple(slice(o, o + e) for o, e in zip(off, loc))
        s = dequant_fp8_oracle.expand(scale.numpy(), tuple(loc), src.g, off[-2], off[-1])
        out[box] = np.where(done[box], out[box], s)
        done[box] = True
    return out


def _quantise(x: np.ndarray, dtype: str, g: str, fmt) -> tuple[np.ndarray, np.ndarray]:
    if dtype == "int8":
        return int8_oracle.quantize(x, g)
    if fmt is not None:
        return ue8m0_oracle.quantize(x, g, 0, 0, fmt)
    return block_fp8_oracle.quantize(x) if g == "block" else scaled_fp8_oracle.quantize(x, g)


def _parts_of(spec: Spec, name: str) -> tuple:
    d = spec.dests[name]
    if d.parts is not None:
        return d.parts
    return (PackedPart(name, tuple(slice(0, e) for e in d.shape), tuple(d.window)),)


def expect(spec: Spec, data: Data) -> dict:
    """{name: (destination tensor, scale tensor or None)} the pull must leave (CPU), sentinels outside every part."""
    out = {}
    for name, d in spec.dests.items():
        parts, route = _parts_of(spec, name), spec.route_of(name)
        names = {p.source for p in parts}
        dest = torch.full((int(np.prod(d.shape)) * DT[d.dtype].itemsize,), SENTINEL, dtype=torch.uint8)
        dest = dest.view(DT[d.dtype]).reshape(d.shape)
        scale = None
        if route in ("copy", "cast", "dequant", "verbatim"):
            srcs = {}
            for n in names:
                src = spec.sources[n]
                srcs[n] = _bits(dequantised(src, data, n, d.dtype) if route == "dequant" else
                                convert(data.full[n], src.dtype, d.dtype))
            dest = _from_bits(packed_oracle.fill(_bits(dest), parts, srcs), d.dtype).reshape(d.shape)
            if route == "verbatim":
                s = packed_oracle.fill(np.zeros(d.shape, np.float32), parts,
                                       {n: scale_of_element(spec.sources[n], data, n) for n in names})
                s = {"block": s[..., ::BLOCK, ::BLOCK], "channel": s[..., :, :1], "tensor": s[..., 0, 0]}[d.g]
                scale = torch.from_numpy(np.ascontiguousarray(s))
        else:
            xs = {}
            for n in names:
                src = spec.sources[n]
                xs[n] = (dequantised(src, data, n, "float32") if route == "requant" else data.full[n].float()).numpy()
            x = packed_oracle.fill(np.zeros(d.shape, np.float32), parts, xs)
            q, s = _quantise(x, d.dtype, d.g, spec.scale_fmt)
            dest = _from_bits(np.ascontiguousarray(q).view(np.uint8 if d.dtype == "e4m3" else np.int8), d.dtype) \
                if d.dtype == "e4m3" else torch.from_numpy(np.ascontiguousarray(q))
            scale = torch.from_numpy(np.ascontiguousarray(s, dtype=np.float32).reshape(
                source_scale_shapes(d.g, d.shape, 0, 0)[0]))
        out[name] = (dest, scale)
    return out


EXACT_ROUTES = ("copy", "verbatim")  # bytes moved as they are: every bit, NaN payloads included, is the contract


def _nan(t: torch.Tensor) -> torch.Tensor:
    if t.dtype in (torch.int8, torch.uint8):
        return torch.zeros(t.shape, dtype=torch.bool)
    return t.float().isnan()


def assert_same(got: torch.Tensor, want: torch.Tensor, what: str, exact: bool = False) -> None:
    """Bit for bit.  Unless ``exact``, NaN equals NaN whatever its bits: on converting routes the oracles' NaN
    patterns are not the contract; on byte moves (``exact``) they are."""
    got, want = got.cpu(), want.cpu()
    assert got.dtype == want.dtype and tuple(got.shape) == tuple(want.shape), (what, got.dtype, want.dtype, got.shape)
    same = _bits(got) == _bits(want)
    if not exact:
        same |= (_nan(got) & _nan(want)).numpy()
    if not same.all():
        bad = np.argwhere(~same)
        i = tuple(int(v) for v in bad[0])
        raise AssertionError(f"{what}: {len(bad)} of {same.size} elements differ, first at {i}: got "
                             f"{_bits(got)[i]:#x} ({got[i].float().item()}), want {_bits(want)[i]:#x} "
                             f"({want[i].float().item()})")


def assert_pull(spec: Spec, got: dict, want: dict, what: str) -> None:
    for name, (d, s) in want.items():
        gd, gs = got[name]
        route = spec.route_of(name)
        assert_same(gd, d, f"{what} '{name}' ({route})", exact=route in EXACT_ROUTES)
        if s is not None:
            assert_same(gs.reshape(s.shape), s, f"{what} '{name}' scale", exact=route == "verbatim")


# ---- host tier -------------------------------------------------------------------------------------------------------
class HostBuffer(helpers.HostBuffer):
    """helpers.HostBuffer that also stands in for ScaledNvlinkBuffer and maps its memory, as the compile reads
    it (``window``, ``scale_window``)."""

    def __init__(self, shard: torch.Tensor, scale=None, granularity=None, row0: int = 0, col0: int = 0):
        super().__init__(shard, shard.shape, shard.dtype)
        self.scale, self.granularity, self.row0, self.col0 = scale, granularity, row0, col0

    def window(self, device) -> StridedMem:
        return StridedMem.from_tensor(self.shard)

    def scale_window(self, device) -> StridedMem:
        return StridedMem.from_tensor(self.scale)


def handles_of(spec: Spec, data: Data, make) -> dict:
    """{source: [RDMAWeightHandle]} with ``make(shard, scale or None, granularity, row0, col0)`` buffers."""
    out = {}
    for name, src in spec.sources.items():
        hs = []
        for k, (off, loc) in enumerate(src.boxes):
            shard_ = region(data.full[name], off, loc).contiguous().clone()
            scale = data.scales[name][k].clone() if src.g is not None else None
            buf = make(shard_, scale, src.g, off[-2], off[-1])
            hs.append(RDMAWeightHandle(buf, TensorSlice(tuple(off), (k,), tuple(src.shape), tuple(loc), (len(src.boxes),)), k))
        out[name] = hs
    return out


def refill(spec: Spec, handles: dict, data: Data, shard_of, scale_of) -> None:
    """Write ``data`` into the existing handles' memory (``shard_of(buffer)``, ``scale_of(buffer)`` tensors)."""
    for name, src in spec.sources.items():
        for k, (h, (off, loc)) in enumerate(zip(handles[name], src.boxes)):
            shard_of(h.rdma_buffer).copy_(region(data.full[name], off, loc))
            if src.g is not None:
                scale_of(h.rdma_buffer).copy_(data.scales[name][k])


def dests_of(spec: Spec, device="cpu") -> tuple[dict, dict, dict]:
    """(destinations full of SENTINEL bytes, {keyword: {name: scale full of SCALE_SENTINEL}}, dest_slices)."""
    dests, scales, slices = {}, {f"{g}_scales": {} for g in ("block", "channel", "tensor")}, {}
    for name, d in spec.dests.items():
        n = int(np.prod(d.shape)) * DT[d.dtype].itemsize
        dests[name] = torch.full((n,), SENTINEL, dtype=torch.uint8, device=device).view(DT[d.dtype]).reshape(d.shape)
        if d.g is not None:
            scales[f"{d.g}_scales"][name] = torch.full(source_scale_shapes(d.g, d.shape, 0, 0)[0], SCALE_SENTINEL,
                                                       device=device)
        if d.window is not None:
            src = spec.sources[name]
            slices[name] = TensorSlice(tuple(d.window), (0,), tuple(src.shape), tuple(d.shape), (1,))
    return dests, scales, slices


@dataclass
class HostRun:
    spec: Spec
    handles: dict
    dests: dict
    scales: dict
    ops: list
    windows: dict        # name -> [(src, dst) StridedMem] in op order of that name
    tables: dict         # "copy" | "block" | "scaled" | "dequant" | "requant" | "verbatim" -> compiled tables
    replays: list        # the replay calls, re-run by replay()
    keep: list

    def replay(self) -> None:
        for fn in self.replays:
            fn()

    def owner(self, addr: int) -> tuple[str, int, tuple]:
        """(source name, handle index, global (row, col)) of the source byte at ``addr``."""
        for name, hs in self.handles.items():
            for k, h in enumerate(hs):
                t = h.rdma_buffer.shard
                lo, n = t.data_ptr(), t.numel() * t.element_size()
                if lo <= addr < lo + n:
                    local = np.unravel_index((addr - lo) // t.element_size(), t.shape)
                    off = h.tensor_slice.offsets
                    return name, k, (int(off[-2] + local[-2]), int(off[-1] + local[-1]))
        raise KeyError(addr)

    def owner_of_buffer(self, buf) -> str:
        return next(n for n, hs in self.handles.items() for h in hs if h.rdma_buffer is buf)

    def dest_row(self, addr: int) -> int:
        for name, t in self.dests.items():
            lo = t.data_ptr()
            if lo <= addr < lo + t.numel() * t.element_size():
                return int(np.unravel_index((addr - lo) // t.element_size(), t.shape)[-2])
        raise KeyError(addr)

    def result(self) -> dict:
        return {n: (d, next((s[n] for s in self.scales.values() if n in s), None)) for n, d in self.dests.items()}


def verdicts(spec: Spec, handles: dict, dests: dict, scales: dict) -> tuple[dict, set]:
    """The package's route verdicts for a spec, the checks ``DirectWeightSyncDest.pull`` makes before building a plan:
    (_check_scales, _check_dequant) over the union of the parts' handles, then _check_packed_rows."""
    parts = DirectWeightSyncDest._check_packed(handles, dests, spec.packed())
    route = _route_handles(handles, parts)
    scaled = DirectWeightSyncDest._check_scales(route, {n: cuda_like(t) for n, t in dests.items()}, scales,
                                                requantize=spec.requantize, verbatim=spec.verbatim)
    scaled = {n: (kw, dests[n], s, r) for n, (kw, _, s, r) in scaled.items()}
    dequant = DirectWeightSyncDest._check_dequant(route, dests, scaled)
    DirectWeightSyncDest._check_packed_rows(parts, dequant, {n for n, (*_, r) in scaled.items() if r == "requantise"})
    return scaled, dequant


def refusal(spec: Spec) -> str | None:
    """The ValueError a pull of ``spec`` must raise before compiling, from the spec alone: a dequantising or
    requantising part whose int index drops the destination's last dim (None when there is none)."""
    for name, d in spec.dests.items():
        route = spec.route_of(name)
        if route not in ("dequant", "requant"):
            continue
        what = "dequantising" if route == "dequant" else "requantising"
        for k, p in enumerate(d.parts or ()):
            if isinstance(p.dest_index[-1], int):
                return (rf"packed destination '{name}' part {k} \(source '{p.source}'\): its int index drops the "
                        rf"destination's last dim, which a {what} pull cannot fill")
    return None


def host_pull(spec: Spec, data: Data) -> HostRun:
    """Plan ``spec`` on host memory and compile it on the routes the package's verdicts choose, split as
    ``DirectWeightSyncDest._compile`` splits a pull; the tables are replayed once before returning.

    This restates _compile's split (verbatim scale windows into the copy plan; per name the requantising, block,
    channel/tensor fp8 and int8 quantising plans, the fp8 and int8 dequantising plans and the copy plan) with the
    host compilers in place of ``Plans.build_*``: a change to that split in _compile must be made here too.  The
    pieces it shares with _compile are the package's own (op_windows, _add_dq_source, _quant_target, _verbatim_rects,
    scale_grid, _lift, _as_grid), and the H100 suite pulls the same specs through _compile itself."""
    handles = handles_of(spec, data, HostBuffer)
    dests, scales, slices = dests_of(spec)
    scaled, dequant = verdicts(spec, handles, dests, scales)
    ops = DirectWeightSyncDest()._build_plan(handles, dests, slices, packed=spec.packed())
    vb = DirectWeightSyncDest._verbatim_rects(ops, scaled)
    requant = {n for n, (*_, r) in scaled.items() if r == "requantise"}
    kind = {n: 0 if n in requant else (1 if kw == "block_scales" else 2) + (2 if _is_int8(d) else 0)
            for n, (kw, d, *_) in scaled.items() if n not in vb}
    copy, dq, quant, windows = [], {}, {}, {}
    for n, rects in vb.items():
        kw, dq_, ds, _ = scaled[n]
        g = kw.removesuffix("_scales")
        dst = _as_grid(StridedMem.from_tensor(ds), scale_grid(g, tuple(dq_.shape), 0, 0))
        for op, si, di in rects:
            buf = op.rdma_buffer
            src = _as_grid(buf.scale_window(0), _lift(scale_grid(g, buf.shape, buf.row0, buf.col0), op.dest_dropped, 1))
            copy.append((src.sub(si), dst.sub(di)))
    for op in ops:
        w = DirectWeightSyncDest.op_windows(op, op.rdma_buffer.window(0))
        windows.setdefault(op.name, []).append(w)
        if op.name in kind:
            q = quant.setdefault(kind[op.name], ([], {}, [], []))
            q[0].append(w)
            if kind[op.name] == 0:
                _add_dq_source(q[1], op, 0)
        elif op.name in dequant:
            pairs, sources = dq.setdefault(op.rdma_buffer.dtype == torch.int8, ([], {}))
            pairs.append(w)
            _add_dq_source(sources, op, 0)
        else:
            copy.append(w)
    for n, (kw, d, s, _) in scaled.items():
        if n in kind:
            quant[kind[n]][2].append(n)
            quant[kind[n]][3].append(_quant_target(kw.removesuffix("_scales"), d, s, n in requant))
    flags, fmt = scale_fmt_flags(spec.scale_fmt), spec.scale_fmt
    tables, replays, keep = {}, [], []
    if copy:
        rects, nr = build_rects(copy)
        table, tiles, info = _native.plan_compile_host(0, rects, nr, 0, 256)
        tables["copy"] = (table, tiles, info)
        keep.append(rects)
        replays.append(lambda table=table, tiles=tiles, units=info.tile_bytes // 16:
                       fp8_oracle.replay_plan(table, tiles, units, nan_mode=1))
    if vb:
        tables["verbatim"] = vb
    for int8_src, (pairs, sources) in sorted(dq.items()):
        rects, nr = build_rects(pairs, dequantise=True)
        arr = _array(_native.make_dq_source_array, [s for _, s in sources.values()])
        tiles = _native.dequant_fp8_compile_host(0, rects, nr, arr, len(sources))
        tables["dequant"] = tiles if "dequant" not in tables else np.concatenate([tables["dequant"], tiles])
        keep += [rects, arr]
        replays.append(lambda tiles=tiles, i8=int8_src: (int8_source_oracle.replay_dequant if i8 else
                                                         dequant_fp8_oracle.replay)(tiles))
    for k, (pairs, sources, names, targets) in sorted(quant.items()):
        int8 = k in (3, 4)
        if k == 0:
            rects, nr = build_rects(pairs)
            for i in range(nr):  # a same-dtype fp8 window is an opaque byte move to build_rects
                rects[i].src_dtype = rects[i].dst_dtype = _native.TSB_F8E4M3
            src_arr = _array(_native.make_dq_source_array, [s for _, s in sources.values()])
            tgt = _array(_native.make_sq_target_array, targets)
            tb = _native.requant_fp8_compile_host(0, rects, nr, src_arr, len(sources), tgt, len(targets), flags)
            keep += [src_arr, tgt]
            tables["requant"] = tb
            replays.append(lambda tb=tb: ue8m0_oracle.replay_requant(*tb, fmt) if fmt else requant_fp8_oracle.replay(*tb))
        elif k in (1, 3):
            rects, nr = build_rects(pairs, quantise=True)
            tgt = _array(_native.make_target_array, targets)
            tb = _native.block_fp8_compile_host(0, rects, nr, tgt, len(targets), flags)
            keep.append(tgt)
            tables["block_int8" if int8 else "block"] = tb
            replays.append(lambda tb=tb, i8=int8: int8_oracle.replay_block(*tb) if i8 else
                           ue8m0_oracle.replay_block(*tb, fmt) if fmt else block_fp8_oracle.replay(*tb))
        else:
            rects, nr = build_rects(pairs, quantise=True)
            tgt = _array(_native.make_sq_target_array, targets)
            tb = _native.scaled_fp8_compile_host(0, rects, nr, tgt, len(targets), flags)
            keep.append(tgt)
            tables["scaled_int8" if int8 else "scaled"] = tb
            replays.append(lambda tb=tb, i8=int8: int8_oracle.replay_scaled(*tb) if i8 else
                           ue8m0_oracle.replay_scaled(*tb, fmt) if fmt else scaled_fp8_oracle.replay(*tb))
        keep.append(rects)
    run = HostRun(spec, handles, dests, {k: v for k, v in scales.items() if v}, ops, windows, tables, replays, keep)
    run.replay()
    return run


def _array(make, items):
    arr = make(max(1, len(items)))
    for i, t in enumerate(items):
        arr[i] = t
    return arr


# ---- random specs ------------------------------------------------------------------------------------------------------
RANDOM_ROUTES = ["copy_bf16", "cast_float32_bfloat16", "cast_bfloat16_e4m3", "cast_float16_e5m2",
                 "quant_fp8_block_bfloat16", "quant_fp8_channel_float16", "quant_fp8_tensor_float32",
                 "quant_ue8m0_block_bfloat16", "quant_int8_block_float16", "quant_int8_channel_bfloat16",
                 "dq_e4m3_block_bfloat16", "dq_e4m3_channel_float32", "dq_int8_block_bfloat16", "dq_int8_tensor_float16",
                 "rq_block_block", "rq_channel_block", "rq_tensor_tensor"]


def _guillotine(rng: random.Random, box: list, depth: int) -> list:
    """Cut ``box`` ((start, stop) per dim) by random axis cuts into at most 2**depth boxes."""
    cuttable = [d for d, (s, t) in enumerate(box) if t - s > 1]
    if depth == 0 or not cuttable or rng.random() < 0.2:
        return [box]
    d = rng.choice(cuttable)
    s, t = box[d]
    c = rng.randrange(s + 1, t)
    a, b = list(box), list(box)
    a[d], b[d] = (s, c), (c, t)
    return _guillotine(rng, a, depth - 1) + _guillotine(rng, b, depth - 1)


def _random_layout(rng: random.Random, shape: tuple) -> tuple:
    kind = rng.choice(["whole", "rows", "cols", "uneven", "mesh", "replicated"])
    if kind == "whole":
        return whole(shape)
    if kind in ("rows", "cols", "uneven"):
        dim = len(shape) - (1 if kind == "cols" else 2) if kind != "uneven" else rng.randrange(len(shape))
        return shard(shape, dim, rng.choice([2, 3, 4]) if kind != "rows" else 2) or whole(shape)
    if kind == "mesh":
        r, c = shape[-2], shape[-1]
        return mesh(shape, len(shape) - 2, (rng.randrange(1, r),) if r > 1 else (), len(shape) - 1,
                    (rng.randrange(1, c),) if c > 1 else ())
    return replicated(shape, len(shape) - 2, 2) or whole(shape)


def random_spec(seed: int) -> Spec:
    """A destination of rank 2 to 4 cut by random guillotine cuts into parts, some addressed by int indices; each
    part reads a source of random global shape holding its box at a random offset, in a random handle layout, along a
    random route."""
    rng = random.Random(seed)
    route = ROUTES[RANDOM_ROUTES[seed % len(RANDOM_ROUTES)]]
    rank = rng.choice([2, 2, 3, 4])
    shape = [rng.choice([1, 2, 3]) for _ in range(rank - 2)] + [rng.randrange(1, 200), rng.randrange(1, 300)]
    boxes = _guillotine(rng, [(0, e) for e in shape], rng.randrange(1, 4))
    scaled = route.kind in ("dequant", "requant")
    parts, sources = [], {}
    for i, box in enumerate(boxes):
        index, ext = [], []
        for d, (s, t) in enumerate(box):
            # an int drops the dim; the source keeps at least 2 dims (the dims kept so far and the ones still to come)
            if t - s == 1 and len(ext) + (rank - d - 1) >= 2 and rng.random() < 0.6:
                index.append(s)
            else:
                index.append(slice(s, t))
                ext.append(t - s)
        gshape = tuple(e + rng.choice([0, 0, rng.randrange(1, 140)]) for e in ext)
        offs = tuple(rng.randrange(0, g - e + 1) for g, e in zip(gshape, ext))
        name = f"p{i}"
        sources[name] = Src(gshape, route.src, route.sg if scaled else None, _random_layout(rng, gshape))
        parts.append(PackedPart(name, tuple(index), offs))
    if route.kind in ("copy", "cast", "dequant") and len(parts) > 1 and rng.random() < 0.3:
        gone = parts.pop(rng.randrange(len(parts)))  # a hole: element-wise routes leave it alone
        del sources[gone.source]
    return Spec(sources, {"w": Dst(tuple(shape), route.out, route.g, tuple(parts))},
                requantize=route.kind == "requant", scale_fmt=route.fmt)

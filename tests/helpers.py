"""Shared helpers for the test-suite: seeded random rectangle workloads that can be materialised on
the CPU (for the C oracle) and on CUDA (for the product), Llama-3 layouts, the host-memory stand-ins,
shards, handles and plans of the pull suites that run without a GPU, and the sources, guarded buffers
and pulls of the GPU suites (nothing here touches CUDA at import time)."""

from __future__ import annotations

import asyncio
import contextlib
import hashlib
import random
import types

import numpy as np
import pytest
import torch

import workloads
from torchstore_b200 import _native
from torchstore_b200.direct_weight_sync import (DirectWeightSyncDest, DirectWeightSyncSource, NvlinkBuffer,
                                                RDMAWeightHandle)
from torchstore_b200.planner import StridedMem, build_rects
from torchstore_b200.transport.types import TensorSlice

SAME_DTYPES = [torch.uint8, torch.int16, torch.bfloat16, torch.float16, torch.int32, torch.float32, torch.int64, torch.float64]
CAST_PAIRS = [
    (torch.float32, torch.bfloat16),
    (torch.float32, torch.float16),
    (torch.bfloat16, torch.float32),
    (torch.float16, torch.float32),
    (torch.bfloat16, torch.float16),
    (torch.float16, torch.bfloat16),
    (torch.float64, torch.float32),
    (torch.float32, torch.float64),
]


def random_bits(shape, dtype: torch.dtype, gen: torch.Generator, finite_only: bool = False) -> torch.Tensor:
    """Tensor of `dtype` filled with random bit patterns (so NaN payloads, denormals, etc. occur)."""
    n = int(np.prod(shape)) if len(shape) else 1
    raw = torch.randint(0, 256, (n * dtype.itemsize,), dtype=torch.uint8, generator=gen)
    t = raw.view(dtype).reshape(shape)
    if finite_only and dtype.is_floating_point:
        t = torch.where(torch.isfinite(t), t, torch.zeros((), dtype=dtype))
    return t.clone()


class RectCase:
    """One (src window, dst window) pair described relative to two base buffers, so the same case
    can be instantiated on any device."""

    def __init__(self, src_base_shape, dst_base_shape, src_dtype, dst_dtype, src_view, dst_view):
        self.src_base_shape = tuple(src_base_shape)
        self.dst_base_shape = tuple(dst_base_shape)
        self.src_dtype = src_dtype
        self.dst_dtype = dst_dtype
        self.src_view = src_view  # callable(base) -> view
        self.dst_view = dst_view


def _rand_window(rng: random.Random, shape, base_pad):
    """Pick a base shape >= shape and a slice window of `shape` inside it."""
    base = [s + rng.choice([0, 0, 1, 3, 8]) if base_pad else s for s in shape]
    starts = [rng.randint(0, b - s) for b, s in zip(base, shape)]
    idx = tuple(slice(a, a + s) for a, s in zip(starts, shape))
    return tuple(base), idx


def random_case(rng: random.Random, cast: bool = False, max_elems: int = 1 << 16) -> RectCase:
    if cast:
        sdt, ddt = rng.choice(CAST_PAIRS)
    else:
        sdt = ddt = rng.choice(SAME_DTYPES)
    ndim = rng.choice([1, 1, 2, 2, 2, 3, 4])
    while True:
        shape = [rng.choice([1, 2, 3, 5, 7, 8, 16, 17, 31, 32, 64, 100, 128, 257, 512, 1000]) for _ in range(ndim)]
        if int(np.prod(shape)) <= max_elems:
            break
    sbase, sidx = _rand_window(rng, shape, rng.random() < 0.7)
    dbase, didx = _rand_window(rng, shape, rng.random() < 0.7)
    s_perm = list(range(ndim))
    d_perm = list(range(ndim))
    if ndim >= 2 and rng.random() < 0.2:
        rng.shuffle(s_perm)
    if ndim >= 2 and rng.random() < 0.15:
        rng.shuffle(d_perm)
    # views: base is allocated in permuted order, then permuted back, then windowed
    def mk(perm, base, idx):
        inv = [perm.index(i) for i in range(len(perm))]
        alloc_shape = tuple(base[p] for p in perm)

        def view(buf):
            return buf.reshape(alloc_shape).permute(*inv)[idx]

        return alloc_shape, view

    s_alloc, s_view = mk(s_perm, sbase, sidx)
    d_alloc, d_view = mk(d_perm, dbase, didx)
    return RectCase(s_alloc, d_alloc, sdt, ddt, s_view, d_view)


# ---- edge-biased workloads ----------------------------------------------------------------------------
# Windows aimed at the copy_rects kernel's boundaries for a given copy tile size (in units): rows of
# exactly k tiles and one unit either side, narrow rects whose row count is not a multiple of their
# rows-per-tile, one-unit rows (magic 0), rows one unit short of a tile, wide rows under several
# strided outer dims, 5-D and 6-D windows, and cast windows on both sides of the vector rule.
VECTOR_CAST_PAIRS = [p for p in CAST_PAIRS if torch.float64 not in p]
EDGE_KINDS = ("wide_exact", "wide_minus", "wide_plus", "narrow_ragged", "unit_row", "tile_minus_one",
              "wide_nd", "deep_nd", "aligned", "cast_vector", "cast_scalar")


def _edge_window(rng: random.Random, shape, itemsize: int, aligned: bool, pad_outer: bool):
    """(base shape, window index) of a window of `shape` whose innermost dim is contiguous and never
    merges with the dim above it.  aligned: the window's start and every row pitch are multiples of
    16 bytes (given a 16-byte aligned base); otherwise the window starts one element off alignment."""
    q = max(1, 16 // itemsize)  # elements per 16 bytes
    if aligned:
        start_in = q * rng.randint(0, 2)
        inner = -(-(start_in + shape[-1] + 1) // q) * q + q * rng.randint(0, 1)
    else:
        start_in = 1
        inner = start_in + shape[-1] + rng.randint(1, 5)
    base, starts = [], []
    for d, s in enumerate(shape[:-1]):
        # pad_outer: one spare row in every outer dim but the outermost, so no two outer dims merge
        pad = (1 if d else rng.choice([0, 1])) if pad_outer else rng.choice([0, 1])
        base.append(s + pad)
        starts.append(rng.randint(0, pad))
    base.append(inner)
    starts.append(start_in)
    return tuple(base), tuple(slice(a, a + s) for a, s in zip(starts, shape))


def _edge_outer(rng: random.Random, rows: int, n_dims: int):
    """Split `rows` over n_dims outer extents (each > 1 where possible, product == rows)."""
    dims = []
    for _ in range(n_dims - 1):
        f = next((d for d in (2, 3, 5, 7) if rows % d == 0 and rows // d > 1), None)
        if f is None:
            break
        dims.append(f)
        rows //= f
    dims.append(rows)
    rng.shuffle(dims)
    return dims


def edge_case(rng: random.Random, tile_units: int, kind: str, uniform: str | None = None) -> RectCase:
    """One window of `kind` (see EDGE_KINDS) for copy tiles of `tile_units` units.

    uniform="b16": a same-dtype window of 16-byte units, so a workload of them compiles to KIND_B16;
    uniform="f32_bf16": a vector fp32->bf16 window, so a workload of them compiles to KIND_F32_BF16."""
    T = tile_units
    if uniform == "b16":
        sdt = ddt = rng.choice(SAME_DTYPES)
        aligned, vec_cast = True, False
    elif uniform == "f32_bf16":
        sdt, ddt = torch.float32, torch.bfloat16
        aligned, vec_cast = True, True
    elif kind == "cast_vector":
        sdt, ddt = rng.choice(VECTOR_CAST_PAIRS)
        aligned, vec_cast = True, True
    elif kind == "cast_scalar":
        sdt, ddt = rng.choice(CAST_PAIRS)
        aligned, vec_cast = False, False
    else:
        sdt = ddt = rng.choice(SAME_DTYPES)
        aligned, vec_cast = kind == "aligned" or rng.random() < 0.5, False
    cast = sdt != ddt
    # elements per unit: 8 for a vector cast, 16 bytes for an aligned byte move, one element otherwise
    epu = 8 if vec_cast else (16 // sdt.itemsize if aligned and not cast else 1)
    units, rows, n_outer = edge_geometry(rng, T, kind)
    outer = _edge_outer(rng, rows, n_outer) if n_outer else []
    if not outer and rows > 1:
        outer = [rows]
    shape = outer + [units * epu]
    pad_outer = kind in ("wide_nd", "deep_nd") or rng.random() < 0.7
    sbase, sidx = _edge_window(rng, shape, sdt.itemsize, aligned, pad_outer)
    dbase, didx = _edge_window(rng, shape, ddt.itemsize, aligned, pad_outer)
    if not aligned and cast and rng.random() < 0.5:
        # misalign only one side: still no vector mode, but the other side is a clean pitch
        dbase, didx = _edge_window(rng, shape, ddt.itemsize, True, pad_outer)
    return RectCase(sbase, dbase, sdt, ddt, lambda b, i=sidx: b[i], lambda b, i=didx: b[i])


def edge_geometry(rng: random.Random, tile_units: int, kind: str):
    """(units per row, rows, outer dims) of a window of `kind` (see EDGE_KINDS) for copy tiles of
    `tile_units` units."""
    T = tile_units
    big = T >= 4096  # keep the largest tile sizes to a few tens of MiB per workload
    n_outer = 0
    if kind in ("wide_exact", "wide_minus", "wide_plus"):
        k = rng.choice([1, 2])
        units = k * T + {"wide_exact": 0, "wide_minus": -1, "wide_plus": 1}[kind]
        rows, n_outer = rng.choice([1, 2, 3]), rng.choice([0, 1, 2])
    elif kind == "narrow_ragged":
        units = rng.choice([max(1, T // 3), max(1, T // 4 + 1), rng.randint(1, 7)])
        split = max(1, T // units)
        if split == 1:
            units, split = max(1, T // 3), max(1, T // max(1, T // 3))
        rows = split * rng.randint(1, 2) + rng.randint(1, max(1, split - 1))
        n_outer = rng.choice([1, 2])
    elif kind == "unit_row":
        units, rows, n_outer = 1, rng.randint(2, 3 * T + 7), rng.choice([1, 2, 3])
    elif kind == "tile_minus_one":
        units, rows, n_outer = T - 1, rng.randint(2, 7), rng.choice([1, 2])
    elif kind == "wide_nd":
        n_outer = rng.randint(2, 3 if big else 5)
        units = T + rng.choice([0, 1, 7] if big else [0, 1, 7, T // 2])
        rows = 2 ** n_outer * (1 if big else rng.choice([1, 1, 3]))
    elif kind == "deep_nd":
        n_outer = rng.choice([4, 5])
        units = rng.choice([1, 3, T // 2, T + 1]) if not big else rng.choice([1, 3, 100])
        rows = 2 ** n_outer * rng.choice([1, 3])
    else:  # aligned / cast_vector / cast_scalar: a random N-D window
        n_outer = rng.choice([0, 1, 2, 3])
        units = rng.choice([1, 2, 5, 31, T // 2, T, T + 3])
        rows = max(1, rng.choice([1, 3, 8, 17]) * max(1, n_outer))
    return max(1, units), rows, n_outer


def edge_workload(rng: random.Random, tile_units: int, uniform: str | None = None, cast: bool | None = None,
                  extra: int = 6) -> list:
    """Every edge kind at least once (casts only where `cast` allows), plus `extra` more, shuffled.
    cast=None mixes copies and casts; uniform= as in edge_case (all windows of one mode)."""
    if uniform is not None or cast is False:
        kinds = [k for k in EDGE_KINDS if not k.startswith("cast")]
    elif cast:
        kinds = [k for k in EDGE_KINDS if k.startswith("cast")] * 3
    else:
        kinds = list(EDGE_KINDS)
    kinds = kinds + [rng.choice(kinds) for _ in range(extra)]
    rng.shuffle(kinds)
    if cast:
        return [edge_case(rng, tile_units, k) for k in kinds] + [
            edge_case(rng, tile_units, k, uniform="f32_bf16") for k in EDGE_KINDS if not k.startswith("cast")]
    return [edge_case(rng, tile_units, k, uniform) for k in kinds]


# ---- compiled plan tables -----------------------------------------------------------------------------
# DevRect (csrc/tsb_internal.h) as a numpy record: 192 bytes per rect of a tsb_plan_compile_host table.
DEV_RECT = np.dtype([
    ("src", "<u8"), ("dst", "<u8"), ("src_stride", "<i8", (6,)), ("dst_stride", "<i8", (6,)), ("ext", "<u4", (6,)),
    ("n_outer", "<u4"), ("rows", "<u4"), ("units_per_row", "<u4"), ("magic", "<u4"), ("wide", "<u4"), ("split", "<u4"),
    ("mode", "<u4"), ("src_unit_bytes", "<u4"), ("dst_unit_bytes", "<u4"), ("tile_units", "<u4"), ("link", "<u4"),
    ("pad_", "<u4", (3,)),
])
assert DEV_RECT.itemsize == 192
MODE_B16, MODE_F32_BF16_V8, MODE_BF16_E4M3_V16 = 4, 8, 26
VECTOR_CAST_MODES = (8, 10, 12, 14, 16, 18)
KIND_GENERIC, KIND_B16, KIND_F32_BF16, KIND_BF16_E4M3 = 0, 1, 2, 3


KNOBS = ("TSB_TILE_BYTES", "TSB_STATIC_SCHED", "TSB_MAX_GRID", "TSB_FORCE_GENERIC", "TSB_LINK", "TSB_LINK_STAGES",
         "TSB_LINK_STAGE_BYTES", "TSB_CTAS_PER_SM")
# A covering design over (tile bytes, grid cap, scheduling, TSB_FORCE_GENERIC, TSB_LINK): every value of
# every axis, and every (tile bytes, grid cap) pair.  Static scheduling only applies to plans without
# link tiles, so it runs with TSB_LINK=1 on local sources.
KERNEL_REGIMES = [
    # tile bytes, grid cap, scheduling, force generic, TSB_LINK
    (1024, None, "dynamic", False, 2),
    (1024, 1, "static", True, 1),
    (1024, 5, "dynamic", False, 1),
    (4096, None, "static", False, 1),
    (4096, 1, "dynamic", True, 2),
    (4096, 5, "static", True, 1),
    (65536, None, "dynamic", True, 1),
    (65536, 1, "dynamic", False, 2),
    (65536, 5, "static", False, 1),
    (524288, None, "static", True, 1),
    (524288, 1, "dynamic", False, 1),
    (524288, 5, "dynamic", True, 2),
]


def set_knobs(monkeypatch, **knobs):
    for k in KNOBS:
        monkeypatch.delenv(k, raising=False)
    for k, v in knobs.items():
        if v is not None:
            monkeypatch.setenv(k, str(v))


def compiled(pairs):
    """(rects, n, rect table fields, host PlanInfo) of `pairs` under the current knobs."""
    rects, n = rects_for(pairs)
    table, _, info = _native.plan_compile_host(0, rects, n, 0, 0)
    return rects, n, rect_fields(table), info


def run_plan(rects, n):
    """Compile, run on torch's stream, wait, destroy; returns the plan's PlanInfo."""
    plan = _native.plan_create(0, rects, n)
    info = _native.plan_info(plan)
    _native.plan_run(plan, _native.torch_stream(0))
    torch.cuda.synchronize()
    _native.plan_destroy(plan)
    return info


def rect_fields(table: np.ndarray) -> np.ndarray:
    """The rect table of _native.plan_compile_host as a record array with DevRect's field names."""
    return np.ascontiguousarray(table).view(DEV_RECT)


def plan_kind(fields: np.ndarray) -> int:
    """The kernel specialisation a plan of these compiled rects launches (plan.cu Compiler::kind)."""
    if len(fields) and (fields["mode"] == MODE_B16).all():
        return KIND_B16
    if len(fields) and (fields["mode"] == MODE_F32_BF16_V8).all():
        return KIND_F32_BF16
    if len(fields) and (fields["mode"] == MODE_BF16_E4M3_V16).all():
        return KIND_BF16_E4M3
    return KIND_GENERIC


def edge_coverage(fields: np.ndarray, tile_units: int) -> dict:
    """Which of the kernel's tile boundaries the copy-queue rects of `fields` (tile size `tile_units`) reach."""
    f = fields[fields["tile_units"] == tile_units]
    T = tile_units
    upr, wide, split, rows, n_outer = (f[k].astype(np.int64) for k in ("units_per_row", "wide", "split", "rows", "n_outer"))
    return {
        "rows_of_k_tiles": bool(((upr % T == 0) & (wide == 1)).any()),
        "rows_of_k_tiles_plus_1": bool(((upr % T == 1) & (wide == 1)).any()),
        "rows_of_k_tiles_minus_1": bool((upr % T == T - 1).any()),
        "narrow_ragged": bool(((wide == 0) & (split > 1) & (rows % np.maximum(split, 1) != 0)).any()),
        "one_unit_rows": bool(((upr == 1) & (f["magic"] == 0)).any()),
        "tile_minus_one_rows": bool(((wide == 0) & (split == 1) & (upr == T - 1)).any()),
        "wide_under_2_outer": bool(((wide == 1) & (n_outer >= 2)).any()),
        "narrow_nd": bool(((wide == 0) & (n_outer >= 2)).any()),
        "outer_4_or_more": bool((n_outer >= 4).any()),
    }


def materialise(cases, device, seed: int, finite_only: bool = False):
    """Allocate bases on `device` (filled from a seeded CPU generator so CPU and CUDA copies hold
    identical bytes) and return [(src_view, dst_view, dst_base)]."""
    gen = torch.Generator().manual_seed(seed)
    out = []
    for c in cases:
        # +2 elements of slack and an optional odd offset exercise unaligned bases
        src_base = random_bits(c.src_base_shape, c.src_dtype, gen, finite_only).to(device)
        dst_base = random_bits(c.dst_base_shape, c.dst_dtype, gen, True).to(device)
        out.append((c.src_view(src_base), c.dst_view(dst_base), dst_base, src_base))
    return out


def rects_for(pairs):
    """[(src_view, dst_view, ...)] -> (ctypes rect array, n)."""
    return build_rects([(StridedMem.from_tensor(p[0]), StridedMem.from_tensor(p[1])) for p in pairs])


def bytes_of(t: torch.Tensor) -> np.ndarray:
    if t.numel() == 0:
        return np.zeros(0, dtype=np.uint8)
    return t.detach().cpu().contiguous().reshape(-1).view(torch.uint8).numpy().copy()


NAN_CHECK = {
    torch.bfloat16: (np.uint16, 0x7F80, 0x007F),
    torch.float16: (np.uint16, 0x7C00, 0x03FF),
    torch.float32: (np.uint32, 0x7F800000, 0x007FFFFF),
    torch.float64: (np.uint64, 0x7FF0000000000000, 0x000FFFFFFFFFFFFF),
}


def assert_equal_modulo_nan(got: torch.Tensor, want: torch.Tensor, cast: bool):
    """Bit-exact; for cast outputs any NaN encoding equals any other NaN (see DESIGN.md)."""
    g, w = bytes_of(got), bytes_of(want)
    if not cast or got.dtype not in NAN_CHECK:
        assert np.array_equal(g, w)
        return
    np_t, emask, mmask = NAN_CHECK[got.dtype]
    gb, wb = g.view(np_t), w.view(np_t)
    gn = ((gb & np_t(emask)) == np_t(emask)) & ((gb & np_t(mmask)) != 0)
    wn = ((wb & np_t(emask)) == np_t(emask)) & ((wb & np_t(mmask)) != 0)
    assert np.array_equal(gn, wn)
    assert np.array_equal(gb[~wn], wb[~wn])


def assert_same_bits_or_nan(got: torch.Tensor, want: torch.Tensor):
    """On the device: equal bits, or both NaN (the assert_equal_modulo_nan rule)."""
    assert got.shape == want.shape and got.dtype == want.dtype
    as_int = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[got.element_size()]
    same = got.view(as_int) == want.view(as_int)
    if got.is_floating_point():
        same |= torch.isnan(got) & torch.isnan(want)
    assert bool(same.all()), int((~same).sum())


# ---- Llama-3 layouts (torchtitan TP plan; SURVEY.md section 8 header) -------------------------------
LLAMA3_8B = dict(dim=4096, n_layers=32, n_heads=32, n_kv_heads=8, vocab=128256, ffn=14336)
LLAMA3_70B = dict(dim=8192, n_layers=80, n_heads=64, n_kv_heads=8, vocab=128256, ffn=28672)


def llama_layout(cfg=LLAMA3_8B, n_layers: int | None = None, scale: int = 1):
    """name -> (global shape, TP placement).  `scale` divides every dimension (small test models)."""
    d = cfg["dim"] // scale
    kv = cfg["dim"] // cfg["n_heads"] * cfg["n_kv_heads"] // scale
    ffn = cfg["ffn"] // scale
    vocab = cfg["vocab"] // scale
    layers = cfg["n_layers"] if n_layers is None else n_layers
    out = {"tok_embeddings.weight": ((vocab, d), ("S", 0))}
    for i in range(layers):
        p = f"layers.{i}."
        out[p + "attention.wq.weight"] = ((d, d), ("S", 0))
        out[p + "attention.wk.weight"] = ((kv, d), ("S", 0))
        out[p + "attention.wv.weight"] = ((kv, d), ("S", 0))
        out[p + "attention.wo.weight"] = ((d, d), ("S", 1))
        out[p + "feed_forward.w1.weight"] = ((ffn, d), ("S", 0))
        out[p + "feed_forward.w2.weight"] = ((d, ffn), ("S", 1))
        out[p + "feed_forward.w3.weight"] = ((ffn, d), ("S", 0))
        out[p + "attention_norm.weight"] = ((d,), ("R",))
        out[p + "ffn_norm.weight"] = ((d,), ("R",))
    out["norm.weight"] = ((d,), ("R",))
    out["output.weight"] = ((vocab, d), ("S", 0))
    return out


# ---- host-side pulls: shards, handles and plans on host memory -----------------------------------------
def shard_box(shape, n, r, dim):
    """(offsets, local shape) of rank r of n torch.chunk-style Shard(dim) shards of `shape` (empty past the end)."""
    return workloads.shard_box(shape, n, r, ("S", dim))


def region(t, off, loc):
    """The box of `t` at offsets `off` with extent `loc`."""
    return t[tuple(slice(o, o + s) for o, s in zip(off, loc))]


def rand_full(shape, dtype, seed):
    """Seeded normal values scaled by powers of two from 2^-6 to 2^5, in `dtype`."""
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * 2.0 ** torch.randint(-6, 6, shape, generator=g).float()).to(dtype)


def sha256_of(t: torch.Tensor) -> str:
    return hashlib.sha256(t.detach().cpu().contiguous().view(torch.uint8).numpy().tobytes()).hexdigest()


class HostBuffer:
    """Host-memory stand-in for NvlinkBuffer: the planner reads ``shape`` and ``dtype`` only; ``shard`` is what
    the tests move (None for metadata-only plans)."""

    def __init__(self, shard, shape, dtype):
        self.shard, self.shape, self.dtype = shard, tuple(shape), dtype


def shard_handles(full, src_boxes, make_buffer):
    """Handles over the `src_boxes` shards of `full`, rank r holding box r (an empty box gets no handle);
    ``make_buffer(shard, offsets, local shape)`` wraps each contiguous shard -> (handles, keepalive)."""
    gshape = tuple(full.shape)
    handles, keep = [], []
    for r, (off, loc) in enumerate(src_boxes):
        if 0 in loc:
            continue
        shard = region(full, off, loc).contiguous()
        keep.append(shard)
        handles.append(RDMAWeightHandle(rdma_buffer=make_buffer(shard, off, loc),
                                        tensor_slice=TensorSlice(off, (r,), gshape, loc, (len(src_boxes),)), source_rank=r))
    return handles, keep


def plan_windows(handles, dest, dst_box):
    """The product's plan of a pull of one tensor's `handles` into `dest`, the tensor's box `dst_box`
    -> (ops, their (source, destination) windows over each buffer's ``shard``)."""
    off, loc = dst_box
    gshape = tuple(handles[0].tensor_slice.global_shape)
    ops = DirectWeightSyncDest()._build_plan({"w": handles}, {"w": dest}, {"w": TensorSlice(off, (0,), gshape, loc, (1,))})
    return ops, [DirectWeightSyncDest.op_windows(op, StridedMem.from_tensor(op.rdma_buffer.shard)) for op in ops]


def fsdp_handles(layout, n: int, make_buffer, names=None) -> dict[str, list]:
    """Every tensor of ``layout`` cut into ``n`` Shard(0) shards: name -> handles in rank order.
    ``make_buffer(name, offsets, local shape)`` creates each handle's buffer."""
    out = {}
    for name, (shape, _) in layout.items():
        if names is not None and name not in names:
            continue
        hs = []
        for r in range(n):
            off, loc = workloads.shard_box(shape, n, r, ("S", 0)) if n > 1 else ((0,) * len(shape), tuple(shape))
            hs.append(RDMAWeightHandle(make_buffer(name, off, loc), TensorSlice(off, (r,), tuple(shape), loc, (n,)), r))
        out[name] = hs
    return out


def handles_of(shape, n=1, dtype=torch.bfloat16, dim=0, sources=None):
    """FSDP(n) handles of one ``shape`` tensor cut along ``dim`` (torch.chunk-style, uneven when n does not divide
    it), over the shards of ``sources``, or metadata-only buffers without."""
    out = []
    for r in range(n):
        off, loc = workloads.shard_box(shape, n, r, ("S", dim)) if n > 1 else ((0,) * len(shape), tuple(shape))
        shard = None if sources is None else region(sources, off, loc).contiguous()
        out.append(RDMAWeightHandle(HostBuffer(shard, loc, dtype), TensorSlice(off, (r,), tuple(shape), loc, (n,)), r))
    return out


def pull_args(vlayout, tp: int, rank: int, make_dest):
    """-> (destination dict, dest_slices, packed) of a vLLM layout; ``make_dest(name, local shape)``."""
    dests, slices, packed = {}, {}, {}
    for name, (shape, parts, box) in vlayout.items():
        dests[name] = make_dest(name, shape)
        if parts is None:
            slices[name] = TensorSlice(box[0], (rank,), box[1], tuple(shape), (tp,))
        else:
            packed[name] = parts
    return dests, slices, packed


def unfused_args(vlayout, hf_layout, tp: int, rank: int, make_dest):
    """The same bytes pulled without packing: one HF-named destination per part (its box, at the part's source
    offsets) plus the unpacked names -> (destination dict, dest_slices, {fused name: [(part, unfused name)]})."""
    dests, slices, where = {}, {}, {}
    for name, (shape, parts, box) in vlayout.items():
        if parts is None:
            dests[name] = make_dest(name, shape)
            slices[name] = TensorSlice(box[0], (rank,), box[1], tuple(shape), (tp,))
            continue
        for k, p in enumerate(parts):
            ext = tuple(torch.empty(shape, device="meta")[p.dest_index].shape)
            uname = p.source if p.source not in dests else f"{p.source}#{k}"
            assert uname == p.source, "one unfused destination per source"
            dests[uname] = make_dest(uname, ext)
            slices[uname] = TensorSlice(tuple(p.source_offsets), (rank,), tuple(hf_layout[p.source][0]), ext, (tp,))
            where.setdefault(name, []).append((p, uname))
    return dests, slices, where


# ---- validation before anything is exported or compiled ------------------------------------------------
def expect_invalid(fn, needle=None):
    """``fn()`` raises TsbError with TSB_ERR_INVALID (and a message matching ``needle``) -> the message."""
    with pytest.raises(_native.TsbError, match=needle) as e:
        fn()
    assert e.value.code == _native.TSB_ERR_INVALID, e.value
    return str(e.value)


def cuda_like(t):
    """A CPU tensor's metadata that claims to be on CUDA (validation reads nothing else)."""
    return types.SimpleNamespace(dtype=t.dtype, shape=t.shape, dim=t.dim, numel=t.numel, is_contiguous=t.is_contiguous,
                                 stride=t.stride, is_cuda=True, device=t.device)


def fake_dest(dtype, shape=(256, 256)):
    """A contiguous 'CUDA' destination stand-in for _check_scales (it reads dtype, shape, contiguity and device)."""
    return types.SimpleNamespace(dtype=dtype, shape=torch.Size(shape), dim=lambda: len(shape), numel=lambda: 256 * 256,
                                 is_contiguous=lambda: True, is_cuda=True, device=torch.device("cpu"), data_ptr=lambda: 0)


def scaled_handle(dtype, granularity=None):
    """A handle whose buffer has ``dtype`` and, when given, a scale ``granularity``: all the route checks read."""
    buf = types.SimpleNamespace(dtype=dtype)
    if granularity:
        buf.granularity = granularity
    return types.SimpleNamespace(rdma_buffer=buf)


class Boom(Exception):
    pass


def _boom(*a, **k):
    raise Boom("exported, allocated or compiled before validation finished")


def no_compile(monkeypatch):
    """Any plan compile during the test raises Boom.  A module binds it as a fixture with
    ``no_compile = pytest.fixture(no_compile)``."""
    import torchstore_b200.direct_weight_sync as dws

    for name in ("build", "build_source_quant", "build_dequant_fp8", "build_requant_fp8", "build_block_fp8",
                 "build_scaled_fp8"):
        monkeypatch.setattr(dws.Plans, name, classmethod(_boom))


def no_export(monkeypatch):
    """Any export, allocation (torch.empty) or plan compile during the test raises Boom.  A module binds it as a
    fixture with ``no_export = pytest.fixture(no_export)``."""
    import torchstore_b200.direct_weight_sync as dws

    monkeypatch.setattr(dws.HbmDescriptor, "from_tensor", staticmethod(_boom))
    monkeypatch.setattr(torch, "empty", _boom)
    no_compile(monkeypatch)


# ---- device suites: sessions, guarded buffers, sources and pulls on the GPU ------------------------------
DEV = "cuda:0"
E4M3 = torch.float8_e4m3fn
I8 = torch.int8
KW = {"block": "block_scales", "channel": "channel_scales", "tensor": "tensor_scales"}
GUARD = 0x5A
LEAD = 256

needs_two_gpus = pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")


def run(coro):
    return asyncio.run(coro)


def native_session():
    """The native library for one module's tests, and every launch finished and cached block freed after them.  A
    module binds it as ``_init = pytest.fixture(scope="module", autouse=True)(native_session)``."""
    _native.init()
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


@contextlib.contextmanager
def named(what):
    """Prefix a failing comparison with the layout it ran on."""
    try:
        yield
    except AssertionError as e:
        raise AssertionError(f"{what}: {e}") from e


def skip_unless_free(nbytes):
    free, _ = torch.cuda.mem_get_info(DEV)
    if free < 3 * nbytes:
        pytest.skip(f"needs {3 * nbytes / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free")


def guarded(shape, dtype, device=DEV):
    """A contiguous tensor of `shape` inside a GUARD-filled byte buffer (LEAD bytes before, LEAD after)
    -> (buffer, tensor)."""
    n = int(np.prod(shape, dtype=np.int64)) * dtype.itemsize
    base = torch.full((n + 2 * LEAD,), GUARD, dtype=torch.uint8, device=device)
    return base, base[LEAD: LEAD + n].view(dtype).view(shape)


def guards_intact(base):
    return bool((base[:LEAD] == GUARD).all()) and bool((base[-LEAD:] == GUARD).all())


def dest_scale_shape(granularity, local_shape):
    """The scale_inv shape of a `granularity`-scaled destination of `local_shape`."""
    *lead, n, k = local_shape
    return {"block": (*lead, -(-n // 128), -(-k // 128)), "channel": (*lead, n, 1), "tensor": tuple(lead)}[granularity]


def register_shards(global_shape, shards, *, name="w", device=DEV, granularity=None, **register_kw):
    """One DirectWeightSyncSource per entry (offsets, shard, scale or None) of `shards`: rank r publishes shard r on
    `device` over its box of `global_shape`, with its scale under KW[granularity]; a None entry keeps its rank and
    publishes nothing -> (sources [(source, device shard, device scale or None)], handles)."""
    sources, handles = [], []
    for r, entry in enumerate(shards):
        if entry is None:
            continue
        off, shard, scale = entry
        shard, kw = shard.to(device), dict(register_kw)
        if scale is not None:
            scale = scale.to(device)
            kw[KW[granularity]] = {name: scale}
        sl = TensorSlice(tuple(off), (r,), tuple(global_shape), tuple(shard.shape), (len(shards),))
        src = DirectWeightSyncSource()
        handles.append(src.register({name: shard}, rank=r, tensor_slices={name: sl}, **kw)[name])
        sources.append((src, shard, scale))
    return sources, handles


def register_boxes(full, boxes, *, scale_of=None, **kw):
    """register_shards of the `boxes` (offsets, local shape) of `full`, rank r holding box r (an empty box publishes
    nothing); ``scale_of(offsets, local shape)`` gives each shard's scale."""
    shards = [None if 0 in loc else (off, region(full, off, loc).contiguous(), scale_of(off, loc) if scale_of else None)
              for off, loc in boxes]
    return register_shards(full.shape, shards, **kw)


def cleanup(sources):
    for source, *_ in sources:
        run(source.cleanup())


def pull_box(handles, full_shape, box, dtype, *, granularity=None, sync=None, device=DEV, name="w", **pull_kw):
    """Pull `handles` into a guarded `dtype` destination over the `box` (offsets, local shape) of the tensor, with a
    guarded float32 scale under KW[granularity] when given (``requantize``, ``scale_fmt`` and ``verbatim`` pass
    through) -> (sync, destination, scale or None, guard buffers)."""
    off, loc = box
    base, y = guarded(loc, dtype, device)
    guards, scale, scales = (base,), None, {}
    if granularity is not None:
        sbase, scale = guarded(dest_scale_shape(granularity, loc), torch.float32, device)
        guards, scales = (base, sbase), {KW[granularity]: {name: scale}}
    sync = sync or DirectWeightSyncDest()
    run(sync.pull({name: handles}, {name: y}, {name: TensorSlice(off, (0,), tuple(full_shape), loc, (1,))}, **scales,
                  **pull_kw))
    return sync, y, scale, guards


# ---- packed destinations on the GPU -------------------------------------------------------------------------
def masters(layout, seed, device=DEV):
    g = torch.Generator(device).manual_seed(seed)
    return {n: (torch.randn(shape, device=device, generator=g) * 0.02).to(torch.bfloat16)
            for n, (shape, _) in layout.items()}


def nv_handles(layout, n, full):
    return fsdp_handles(layout, n, lambda name, off, loc: NvlinkBuffer(region(full[name], off, loc).contiguous()))


def as_np(t):
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32}[t.element_size()]).cpu().numpy()


def whole_handle(t):
    """One handle over the whole of ``t``."""
    z = (0,) * t.dim()
    return [RDMAWeightHandle(NvlinkBuffer(t.contiguous()), TensorSlice(z, (0,), tuple(t.shape), tuple(t.shape), (1,)), 0)]


def pull(handles, dests, slices=None, **kw):
    sync = DirectWeightSyncDest()
    run(sync.pull(handles, dests, slices, **kw))
    return sync

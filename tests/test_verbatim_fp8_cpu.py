"""Verbatim pulls without a GPU: the scale mapping (verbatim_scale_rects, reached through the planner) applied to
numpy arrays against the group-by-group oracle over a table of layouts and seeded random meshes, its refusals
naming the oracle's first offending group, and the validation of pull(verbatim=True) before anything is
compiled."""

import asyncio
import itertools
import random
import types

import numpy as np
import pytest
import torch

from oracle import reshard_oracle as ro
from oracle.verbatim_fp8_oracle import verbatim
from tests.helpers import Boom, cuda_like, no_export
from torchstore_b200.direct_weight_sync import (DirectWeightSyncDest, RDMAWeightHandle, scale_grid, source_scale_shapes,
                                                verbatim_scale_rects)
from torchstore_b200.transport.types import TensorSlice

E4M3 = torch.float8_e4m3fn
GRANULARITIES = ("block", "channel", "tensor")
KW = {g: f"{g}_scales" for g in GRANULARITIES}


def rows(shape, n, dim=0, lead=0):
    """Boxes of `shape` cut into n even chunks along dim `lead + dim` (the last chunks may be short or empty)."""
    d = lead + dim
    chunk = -(-shape[d] // n)
    out = []
    for r in range(n):
        off, loc = [0] * len(shape), list(shape)
        off[d], loc[d] = min(shape[d], r * chunk), max(0, min(shape[d], (r + 1) * chunk) - r * chunk)
        out.append((tuple(off), tuple(loc)))
    return out


def mesh(shape, nr, nc):
    """A 2-D mesh: nr row chunks x nc column chunks of a 2-D `shape`."""
    return [((r0[0], c0[1]), (rl[0], cl[1])) for (r0, rl), (c0, cl) in itertools.product(rows(shape, nr, 0), rows(shape, nc, 1))]


# (name, global shape, source boxes, destination box, granularities that line up)
LAYOUTS = [
    ("fsdp_rows_to_tp_cols", (512, 640), rows((512, 640), 4), rows((512, 640), 5, 1)[2], {"block", "channel"}),
    ("tp_cols_to_fsdp_rows", (512, 640), rows((512, 640), 5, 1), rows((512, 640), 4)[1], {"block"}),
    ("fsdp_rows_to_tp_rows", (512, 640), rows((512, 640), 4), rows((512, 640), 2)[1], {"block", "channel"}),
    ("mesh_2d", (384, 512), mesh((384, 512), 3, 2), ((128, 256), (256, 256)), {"block", "channel"}),
    ("mesh_2d_to_mesh_2d", (384, 512), mesh((384, 512), 3, 2), ((128, 256), (128, 256)), set(GRANULARITIES)),
    ("replicated", (256, 384), rows((256, 384), 2) * 2, ((0, 0), (256, 384)), {"block", "channel"}),
    ("replicated_exact", (256, 384), rows((256, 384), 2) * 2, ((128, 0), (128, 384)), set(GRANULARITIES)),
    ("moe_experts", (4, 256, 384), rows((4, 256, 384), 2), ((1, 0, 0), (2, 256, 384)), set(GRANULARITIES)),
    ("moe_experts_to_tp", (4, 256, 384), rows((4, 256, 384), 2), ((0, 0, 128), (4, 256, 128)), set(GRANULARITIES)),
    ("moe_rows_to_tp", (3, 256, 384), rows((3, 256, 384), 2, 0, 1), ((0, 0, 256), (3, 256, 128)), {"block", "channel"}),
    ("ragged_tails", (300, 200), [((0, 0), (128, 200)), ((128, 0), (128, 200)), ((256, 0), (44, 200))],
     ((0, 128), (300, 72)), {"block", "channel"}),
    ("ragged_full", (300, 200), [((0, 0), (256, 200)), ((256, 0), (44, 200))], ((0, 0), (300, 200)), {"block", "channel"}),
    ("one_row_shards", (5, 257), rows((5, 257), 5), ((0, 0), (5, 257)), {"channel"}),
    ("one_row_dest", (5, 257), rows((5, 257), 5), ((2, 0), (1, 257)), set(GRANULARITIES)),
    ("one_column_shards", (64, 6), rows((64, 6), 6, 1), ((0, 0), (64, 6)), set()),
    ("one_column_dest", (64, 6), rows((64, 6), 6, 1), ((0, 3), (64, 1)), set(GRANULARITIES)),
    ("single_block_unaligned", (512, 512), rows((512, 512), 4), ((200, 300), (50, 60)), set(GRANULARITIES)),
    # refusals
    ("misaligned_tp_offset", (256, 768), rows((256, 768), 2), rows((256, 768), 4, 1)[1], {"channel"}),
    ("fsdp_cut_inside_block", (300, 256), rows((300, 256), 3), ((0, 0), (300, 256)), {"channel"}),
    ("row_split_across_column_shards", (256, 512), rows((256, 512), 4, 1), ((0, 0), (128, 512)), {"block"}),
    ("tensor_across_two_shards", (256, 256), rows((256, 256), 2), ((64, 0), (128, 256)), {"channel"}),
]


class FakeScaledBuffer:
    """Host-memory stand-in for ScaledNvlinkBuffer (the planner reads these attributes only)."""

    def __init__(self, shard, scale, g, r0, c0):
        self.shard, self.scale, self.granularity, self.row0, self.col0 = shard, scale, g, r0, c0
        self.dtype, self.shape = shard.dtype, tuple(shard.shape)


def fp8_full(shape, seed):
    return torch.from_numpy(np.random.default_rng(seed).integers(0, 256, size=shape, dtype=np.uint8)).view(E4M3)


def shard_scale(g, loc, off, rng):
    """A float32 scale of its own for one shard, in a published shape (per tensor: `lead` or `lead + (1,)`)."""
    shapes = source_scale_shapes(g, loc, off[-2], off[-1])
    return torch.from_numpy(rng.standard_normal(shapes[rng.integers(len(shapes))]).astype(np.float32))


def make_sources(g, q_full, boxes, seed):
    """-> [(shard, scale, offset)] for every non-empty box, each shard with its own scale."""
    rng = np.random.default_rng(seed)
    out = []
    for off, loc in boxes:
        if 0 in loc:
            continue
        shard = q_full[tuple(slice(o, o + e) for o, e in zip(off, loc))].contiguous()
        out.append((shard, shard_scale(g, loc, off, rng), off))
    return out


def plan(g, gshape, sources, dst_box):
    """The product's plan of a verbatim pull of `sources` into `dst_box` -> (ops, dest, dest scale)."""
    handles = [RDMAWeightHandle(rdma_buffer=FakeScaledBuffer(s, sc, g, off[-2], off[-1]), source_rank=r,
                                tensor_slice=TensorSlice(off, (r,), gshape, tuple(s.shape), (len(sources),)))
               for r, (s, sc, off) in enumerate(sources)]
    off, loc = dst_box
    dest = torch.full(loc, 0x55, dtype=torch.uint8).view(E4M3)
    dest_scale = torch.full(source_scale_shapes(g, loc, 0, 0)[0], -7.0)
    ops = DirectWeightSyncDest()._build_plan({"w": handles}, {"w": dest}, {"w": TensorSlice(off, (0,), gshape, loc, (1,))})
    return ops, dest, dest_scale


def apply(g, ops, rects, dest, dest_scale):
    """Move the bytes of every op and the scale rectangles into `dest` / `dest_scale` as the copy plan would;
    every destination scale must be written exactly once."""
    for op in ops:
        src = op.rdma_buffer.shard
        if op.dest_slices is None:
            dest.view(torch.uint8).copy_(src.view(torch.uint8))
        else:
            dest.view(torch.uint8)[op.dest_slices] = src.view(torch.uint8)[op.src_slices]
    grid = scale_grid(g, tuple(dest.shape), 0, 0)
    out = dest_scale.reshape(grid)
    hits = torch.zeros(grid, dtype=torch.int64)
    for op, src_idx, dst_idx in rects:
        buf = op.rdma_buffer
        out[dst_idx] = buf.scale.reshape(scale_grid(g, buf.shape, buf.row0, buf.col0))[src_idx]
        hits[dst_idx] += 1
    assert (hits == 1).all()


def group_text(g, group):
    return {"block": f"block {group}", "channel": f"row {group[:-1]}", "tensor": f"matrix {group[:-2]}"}[g]


def run_layout(g, gshape, sources, dst_box):
    """Plan, map and apply a verbatim pull and compare with the oracle -> whether the groups line up."""
    want_q, want_s, group = verbatim(g, [(s.view(torch.uint8).numpy(), sc.numpy(), off) for s, sc, off in sources], *dst_box)
    ops, dest, dest_scale = plan(g, gshape, sources, dst_box)
    scaled = {"w": (KW[g], dest, dest_scale, "verbatim")}
    if group is not None:
        with pytest.raises(ValueError, match="verbatim pull of 'w'") as e:
            DirectWeightSyncDest._verbatim_rects(ops, scaled)
        assert f"destination {group_text(g, group)} " in str(e.value)
        assert "requantize=True" in str(e.value)
        return False
    rects = DirectWeightSyncDest._verbatim_rects(ops, scaled)["w"]
    apply(g, ops, rects, dest, dest_scale)
    assert np.array_equal(dest.view(torch.uint8).numpy(), want_q)
    assert np.array_equal(dest_scale.numpy().reshape(-1).view(np.uint32), want_s.reshape(-1).view(np.uint32))
    return True


@pytest.mark.parametrize("g", GRANULARITIES)
@pytest.mark.parametrize("name,gshape,boxes,dst_box,lines_up", LAYOUTS, ids=[entry[0] for entry in LAYOUTS])
def test_layout_table_against_the_oracle(g, name, gshape, boxes, dst_box, lines_up):
    q = fp8_full(gshape, len(name))
    assert run_layout(g, gshape, make_sources(g, q, boxes, len(name) + 1), dst_box) == (g in lines_up)


def test_refusals_name_the_oracles_first_group():
    """The pure function returns the same first offending group as the oracle (lead + (group row, group col))."""
    cases = [("block", "misaligned_tp_offset", (0, 0)), ("block", "fsdp_cut_inside_block", (0, 0)),
             ("channel", "row_split_across_column_shards", (0, 0)), ("tensor", "tensor_across_two_shards", (0, 0)),
             ("block", "one_row_shards", (0, 0)), ("channel", "one_column_shards", (0, 0))]
    table = {entry[0]: entry[1:] for entry in LAYOUTS}
    for g, name, first in cases:
        gshape, boxes, dst_box, _ = table[name]
        sources = make_sources(g, fp8_full(gshape, 1), boxes, 2)
        _, _, want = verbatim(g, [(s.view(torch.uint8).numpy(), sc.numpy(), off) for s, sc, off in sources], *dst_box)
        ops, dest, _ = plan(g, gshape, sources, dst_box)
        dst_off = ops[0].dest_offsets
        rects = [(tuple(op.rdma_buffer.shape), op.src_offsets,
                  tuple(zip(*[(o + (s.start if op.dest_slices else 0), (s.stop - s.start) if op.dest_slices else e)
                              for o, s, e in zip(dst_off, op.dest_slices or [None] * dest.dim(), dest.shape)])))
                 for op in ops]
        got, group = verbatim_scale_rects(g, tuple(dest.shape), dst_off, rects)
        assert got == [] and group == want == first, (g, name)


def test_later_offending_groups():
    """The first group is the lexicographically smallest one, also away from the origin."""
    # rows cut at 200, inside block row 1: blocks (1, *) straddle two handles
    q = fp8_full((384, 256), 3)
    sources = make_sources("block", q, [((0, 0), (200, 256)), ((200, 0), (184, 256))], 4)
    box = ((0, 0), (384, 256))
    _, _, want = verbatim("block", [(s.view(torch.uint8).numpy(), sc.numpy(), off) for s, sc, off in sources], *box)
    assert want == (1, 0)
    assert not run_layout("block", (384, 256), sources, box)
    # an MoE stack whose expert 2 alone is cut into two row shards: the destination's matrix (1,) straddles
    q3 = fp8_full((3, 64, 64), 5)
    boxes = [((0, 0, 0), (2, 64, 64)), ((2, 0, 0), (1, 32, 64)), ((2, 32, 0), (1, 32, 64))]
    sources = make_sources("tensor", q3, boxes, 6)
    box = ((1, 0, 0), (2, 64, 64))
    _, _, want = verbatim("tensor", [(s.view(torch.uint8).numpy(), sc.numpy(), off) for s, sc, off in sources], *box)
    assert want == (1, 0, 0)
    assert not run_layout("tensor", (3, 64, 64), sources, box)


def test_coverage_is_checked_on_the_host():
    q = fp8_full((256, 256), 7)
    g = "block"
    # a gap: rows 128..256 are covered by no handle
    sources = make_sources(g, q, [((0, 0), (128, 256))], 8)
    ops, dest, ds = plan(g, (256, 256), sources, ((0, 0), (256, 256)))
    with pytest.raises(ValueError, match="32768 of its 65536 elements are covered by no handle"):
        DirectWeightSyncDest._verbatim_rects(ops, {"w": (KW[g], dest, ds, "verbatim")})
    # two handles over rows 64..128 (partially overlapping replicas): the first element covered twice is named
    sources = make_sources(g, q, [((0, 0), (128, 256)), ((64, 0), (192, 256))], 9)
    ops, dest, ds = plan(g, (256, 256), sources, ((0, 0), (256, 256)))
    with pytest.raises(ValueError, match=r"global element \(64, 0\) is covered by two handles"):
        DirectWeightSyncDest._verbatim_rects(ops, {"w": (KW[g], dest, ds, "verbatim")})
    with pytest.raises(ValueError):
        verbatim(g, [(s.view(torch.uint8).numpy(), sc.numpy(), off) for s, sc, off in sources], (0, 0), (256, 256))
    # no handle reaches the destination at all
    ops, dest, ds = plan(g, (256, 256), make_sources(g, q, [((0, 0), (128, 256))], 8), ((128, 0), (128, 256)))
    with pytest.raises(ValueError, match="no handle covers"):
        DirectWeightSyncDest._verbatim_rects(ops, {"w": (KW[g], dest, ds, "verbatim")})


def rand_layout(rng, ndim):
    md = rng.choice([1, 1, 2])
    shape = tuple(rng.choice([1, 2, 3, 4]) for _ in range(md))
    pl = [rng.choice([("R",)] + [("S", d) for d in range(ndim)]) for _ in range(md)]
    return shape, pl


@pytest.mark.parametrize("seed", range(6))
def test_random_layouts(seed):
    """Seeded random meshes and placements on both sides, 2-D and MoE-like 3-D shapes whose dims are often
    multiples of 128: the product and the oracle agree on every layout, lined up or not."""
    rng = random.Random(9100 + seed)
    lined_up = 0
    for _ in range(12):
        ndim = rng.choice([2, 2, 3])
        dims = [rng.choice([128, 256, 384, 512, 200, 96, 1, 7]) for _ in range(2)]
        gshape = tuple([rng.choice([1, 2, 4])] * (ndim - 2) + dims)
        g = rng.choice(GRANULARITIES)
        q = fp8_full(gshape, seed)
        smesh, spl = rand_layout(rng, ndim)
        dmesh, dpl = rand_layout(rng, ndim)
        boxes = []
        for coord in itertools.product(*(range(m) for m in smesh)):
            sl = ro.make_slice(gshape, smesh, coord, spl)
            boxes.append((tuple(sl.offsets), tuple(sl.local_shape)))
        sources = make_sources(g, q, boxes, seed)
        for coord in itertools.product(*(range(m) for m in dmesh)):
            dsl = ro.make_slice(gshape, dmesh, coord, dpl)
            if 0 in dsl.local_shape:
                continue
            lined_up += run_layout(g, gshape, sources, (tuple(dsl.offsets), tuple(dsl.local_shape)))
    assert lined_up > 0


# ---- pull validation (before anything is compiled) --------------------------------------------------
no_export = pytest.fixture(no_export)


def handles(kinds, dtype=E4M3):
    return [RDMAWeightHandle(rdma_buffer=types.SimpleNamespace(granularity=k, dtype=dtype), source_rank=r,
                             tensor_slice=TensorSlice((0, 0), (r,), (8, 8), (8, 8), (2,))) for r, k in enumerate(kinds)]


def test_route_decision(no_export):
    check = DirectWeightSyncDest._check_scales
    dest = {"w": cuda_like(torch.zeros(8, 8, dtype=E4M3))}
    bs = {"block_scales": {"w": torch.zeros(1, 1)}}
    assert check({"w": handles(["block", "block"])}, dest, bs, verbatim=True)["w"][3] == "verbatim"
    assert check({"w": handles(["block"])}, dest, bs, requantize=True)["w"][3] == "requantise"
    # bf16 handles are still quantised with the flag
    assert check({"w": handles([None], torch.bfloat16)}, dest, bs, verbatim=True)["w"][3] == "quantise"
    with pytest.raises(ValueError, match="exclusive"):
        check({"w": handles(["block"])}, dest, bs, requantize=True, verbatim=True)
    with pytest.raises(ValueError, match="channel-scaled handles.*requantize=True"):
        check({"w": handles(["channel"])}, dest, bs, verbatim=True)
    with pytest.raises(ValueError, match="block/tensor-scaled handles.*requantize=True"):
        check({"w": handles(["block", "tensor"])}, dest, {"tensor_scales": {"w": torch.zeros(())}}, verbatim=True)
    with pytest.raises(TypeError, match="mix scaled fp8 and unscaled sources \\(verbatim=True\\)"):
        check({"w": handles(["block", None])}, dest, bs, verbatim=True)
    with pytest.raises(TypeError, match="bf16, f16 or f32 handles.*verbatim=True reads scaled fp8 handles"):
        check({"w": handles([None])}, dest, bs, verbatim=True)
    # without the flag the default refusal stands
    with pytest.raises(TypeError, match="requantised only with requantize=True"):
        check({"w": handles(["block"])}, dest, bs)


def test_pull_errors_raise_before_compile(no_export):
    dest = {"w": cuda_like(torch.zeros(8, 8, dtype=E4M3))}
    cs = {"w": torch.zeros(8, 1)}
    with pytest.raises(ValueError, match="exclusive"):
        asyncio.run(DirectWeightSyncDest().pull({"w": handles(["channel"])}, dest, channel_scales=cs, requantize=True,
                                                verbatim=True))
    with pytest.raises(ValueError, match="scale_fmt does nothing here"):
        asyncio.run(DirectWeightSyncDest().pull({"w": handles(["channel"])}, dest, channel_scales=cs, verbatim=True,
                                                scale_fmt="ue8m0"))
    with pytest.raises(ValueError, match="requantize=True to convert"):
        asyncio.run(DirectWeightSyncDest().pull({"w": handles(["tensor"])}, dest, channel_scales=cs, verbatim=True))


def test_plan_cache_key_includes_the_flag():
    """A cached plan built without verbatim=True is dropped when the flag is set, and vice versa."""
    for built, flag in ((False, True), (True, False)):
        d = DirectWeightSyncDest()
        d._plan = []
        d._plan_key = (frozenset({("w", "block_scales")}), False, None, built)
        d.close = lambda: (_ for _ in ()).throw(Boom("rebuilt"))
        with pytest.raises(Boom):
            asyncio.run(d.pull({}, {}, block_scales={"w": torch.zeros(1, 1)}, verbatim=flag))


def test_store_path_refuses_the_flag():
    from torchstore_b200 import state_dict_utils

    with pytest.raises(NotImplementedError, match="verbatim needs direct_rdma=True"):
        asyncio.run(state_dict_utils.get_state_dict(None, "k", {"w": torch.zeros(1)}, direct_rdma=False, verbatim=True))


def test_public_signatures_default_to_off():
    import inspect

    from torchstore_b200 import api, state_dict_utils

    for fn in (DirectWeightSyncDest.pull, api.get_state_dict, state_dict_utils.get_state_dict):
        assert inspect.signature(fn).parameters["verbatim"].default is False, fn
    assert inspect.signature(DirectWeightSyncDest.pull).parameters["verbatim"].kind == inspect.Parameter.KEYWORD_ONLY

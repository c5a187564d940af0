"""Packed destinations without a GPU: the validation of ``packed`` before anything is compiled, its keyword on
every public entry point, the planned ops of Llama-3-8B's vLLM TP8 layout from HF FSDP(8) handles against the
numpy oracle of the element rule, the compiled copy plan replayed by the C oracle, and the verbatim scale mapping
of packed block- and channel-scaled destinations."""

import asyncio
import inspect

import numpy as np
import pytest
import torch

import workloads
from oracle import c_oracle
from oracle import packed_oracle as po
from tests.helpers import HostBuffer, fsdp_handles, handles_of, pull_args, region, unfused_args
from torchstore_b200 import _native, api, state_dict_utils
from torchstore_b200.direct_weight_sync import (DirectWeightSyncDest, PackedPart, RDMAWeightHandle, scale_grid,
                                                source_scale_shapes)
from torchstore_b200.planner import StridedMem, build_rects
from torchstore_b200.transport.types import TensorSlice

E4M3 = torch.float8_e4m3fn


def check(dest_shape, packed, handles, match, dests=None):
    dests = dests or {"fused": torch.zeros(dest_shape, dtype=torch.bfloat16)}
    with pytest.raises(ValueError, match=match):
        DirectWeightSyncDest._check_packed(handles, dests, packed)
    # pull() raises the same before anything is compiled
    with pytest.raises(ValueError, match=match):
        asyncio.run(DirectWeightSyncDest().pull(handles, dests, packed=packed))


def P(source, index, offsets):
    return PackedPart(source, index, offsets)


# -- validation ------------------------------------------------------------------------------------------------
def test_unknown_destination():
    check((8, 4), {"nope": (P("a", (slice(0, 8), slice(0, 4)), (0, 0)),)}, {"a": handles_of((8, 4))},
          "packed names 'nope', which is not in the destination state dict")


def test_source_without_handles():
    check((8, 4), {"fused": (P("a", (slice(0, 4), slice(0, 4)), (0, 0)), P("b", (slice(4, 8), slice(0, 4)), (0, 0)))},
          {"a": handles_of((4, 4))}, r"packed destination 'fused' part 1 \(source 'b'\): the source has no handles")


def test_destination_with_handles_of_its_own():
    check((8, 4), {"fused": (P("a", (slice(0, 8), slice(0, 4)), (0, 0)),)},
          {"a": handles_of((8, 4)), "fused": handles_of((8, 4))}, "'fused' also has handles of its own name")


@pytest.mark.parametrize("index,match", [
    ((slice(0, 4), slice(0, 4), slice(0, 1)), "dest_index has 3 entries for a 2-dim destination"),
    ((slice(0, 4),), "dest_index has 1 entries for a 2-dim destination"),
    ((slice(0, 4, 2), slice(0, 4)), r"entry 0 \(slice\(0, 4, 2\)\) has a non-unit step"),
    ((slice(6, 10), slice(0, 4)), r"entry 0 \(slice\(6, 10, None\)\) is out of range"),
    ((slice(-2, 4), slice(0, 4)), "entry 0 .* is out of range"),
    ((slice(3, 3), slice(0, 4)), "entry 0 .* is out of range \\(or empty\\)"),
    ((8, slice(0, 4)), r"entry 0 \(8\) is out of range for extent 8"),
    ((-1, slice(0, 4)), r"entry 0 \(-1\) is out of range"),
    (("0", slice(0, 4)), "entry 0 is a str, not an int or a slice"),
])
def test_bad_index(index, match):
    check((8, 4), {"fused": (P("a", index, (0, 0)),)}, {"a": handles_of((8, 4))},
          r"packed destination 'fused' part 0 \(source 'a'\): (dest_index )?" + match)


def test_box_rank_must_match_the_source():
    # an int entry drops a dim: a 1-dim box cannot read a 2-dim source, and the offsets need the source's rank
    check((8, 4), {"fused": (P("a", (0, slice(0, 4)), (0, 0)),)}, {"a": handles_of((8, 4))},
          "a 1-dim box with 2 source offsets does not match the source's 2-dim global shape")
    check((8, 4), {"fused": (P("a", (slice(0, 8), slice(0, 4)), (0,)),)}, {"a": handles_of((8, 4))},
          "a 2-dim box with 1 source offsets does not match")


def test_source_box_leaves_the_source():
    check((8, 4), {"fused": (P("a", (slice(0, 8), slice(0, 4)), (2, 0)),)}, {"a": handles_of((8, 4))},
          r"part 0 \(source 'a'\): the source box at \(2, 0\) with extent \(8, 4\) leaves the source's global shape \(8, 4\)")
    check((8, 4), {"fused": (P("a", (slice(0, 8), slice(0, 4)), (0, -1)),)}, {"a": handles_of((8, 4))}, "leaves")
    check((8, 4), {"fused": (P("a", (slice(0, 8), slice(0, 4)), (0, 0.0)),)}, {"a": handles_of((8, 4))},
          r"source_offsets \(0, 0.0\) must be ints")


def test_overlapping_parts():
    check((8, 4), {"fused": (P("a", (slice(0, 5), slice(0, 4)), (0, 0)), P("b", (slice(4, 8), slice(0, 4)), (0, 0)))},
          {"a": handles_of((8, 4)), "b": handles_of((8, 4))}, r"part 1 \(source 'b'\): its box overlaps part 0's")
    check((2, 8, 4), {"fused": (P("a", (1, slice(0, 8), slice(0, 4)), (0, 0)), P("b", (slice(1, 2), slice(0, 2), slice(0, 4)), (0, 0, 0)))},
          {"a": handles_of((8, 4)), "b": handles_of((1, 8, 4))}, "part 1 .* overlaps part 0's",
          dests={"fused": torch.zeros(2, 8, 4)})


def test_part_not_covered_names_the_first_hole():
    # rows 4..7 of the source have no handle (shard 1 of 2 is missing): the first uncovered element is (4, 0)
    hs = handles_of((8, 4), n=2)[:1]
    check((8, 4), {"fused": (P("a", (slice(0, 8), slice(0, 4)), (0, 0)),)}, {"a": hs},
          r"part 0 \(source 'a'\): no handle covers global element \(4, 0\) of the source")
    # a 2-D mesh with one tile missing: the first hole is that tile's corner inside the part's box
    mesh = [((0, 0), (4, 4)), ((0, 4), (4, 4)), ((4, 0), (4, 4))]
    hs = [RDMAWeightHandle(HostBuffer(None, loc, torch.bfloat16), TensorSlice(off, (r,), (8, 8), loc, (4,)), r)
          for r, (off, loc) in enumerate(mesh)]
    check((6, 6), {"fused": (P("a", (slice(0, 6), slice(0, 6)), (1, 1)),)}, {"a": hs},
          r"no handle covers global element \(4, 4\)")


def test_values_must_be_tuples_of_packed_parts():
    hs = {"a": handles_of((8, 4))}
    dests = {"fused": torch.zeros(8, 4, dtype=torch.bfloat16)}
    part = P("a", (slice(0, 8), slice(0, 4)), (0, 0))
    for bad in ([part], part, (("a", (slice(0, 8), slice(0, 4)), (0, 0)),)):
        with pytest.raises(TypeError, match=r"packed\['fused'\] must be a tuple of PackedPart"):
            asyncio.run(DirectWeightSyncDest().pull(hs, dests, packed={"fused": bad}))
    with pytest.raises(TypeError, match="dest_index and source_offsets of a PackedPart must be tuples"):
        asyncio.run(DirectWeightSyncDest().pull(hs, dests, packed={"fused": (P("a", [slice(0, 8), slice(0, 4)], (0, 0)),)}))


def test_store_path_refuses_packed():
    with pytest.raises(NotImplementedError, match="packed needs direct_rdma=True"):
        asyncio.run(state_dict_utils.get_state_dict(None, "k", {"w": torch.zeros(4, 4)},
                                                    packed={"w": (P("a", (slice(0, 4), slice(0, 4)), (0, 0)),)}))


def test_packed_is_keyword_only_with_a_none_default():
    for fn in (DirectWeightSyncDest.pull, state_dict_utils.get_state_dict, api.get_state_dict):
        p = inspect.signature(fn).parameters["packed"]
        assert p.kind is inspect.Parameter.KEYWORD_ONLY and p.default is None, fn
    import torchstore_b200 as ts

    assert ts.PackedPart is PackedPart and "PackedPart" in ts.__all__
    with pytest.raises(Exception):
        P("a", (0,), (0,)).source = "b"  # frozen


def test_all_gather_votes_no_for_packed(monkeypatch):
    """The NCCL all-gather fills tensors from shards of their own names: a packed pull never takes it."""
    votes = []
    monkeypatch.setattr(state_dict_utils.dist, "is_initialized", lambda: True)
    monkeypatch.setattr(state_dict_utils.dist, "get_world_size", lambda: 2)
    monkeypatch.setattr(state_dict_utils.dist, "get_rank", lambda: 0)
    monkeypatch.setattr(state_dict_utils.dist, "all_reduce", lambda t, op=None: votes.append(int(t.item())))
    cache = state_dict_utils._DirectRDMACache()
    assert not state_dict_utils._try_all_gather(cache, "k", {"w": torch.zeros(4, 4)}, packed=True)
    assert votes == [0]


# -- planning Llama-3-8B TP8 against the oracle --------------------------------------------------------------------
def apply_ops(ops, dests):
    """Move every op's source window into its destination as the copy plan would (host tensors)."""
    for op in ops:
        src = op.rdma_buffer.shard
        if op.dest_tensor is None:
            op.dest_local.copy_(src.reshape(op.dest_local.shape))
        else:
            box = op.dest_local[op.dest_slices]
            box.copy_(src[op.src_slices].reshape(box.shape))


def host_sources(layout, names, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    return {n: torch.randint(-2 ** 15, 2 ** 15, layout[n][0], generator=g, dtype=torch.int16).view(dtype)
            if dtype.itemsize == 2 else torch.randint(0, 256, layout[n][0], generator=g, dtype=torch.uint8)
            for n in names}


def plan_layout(hf, vl, tp, rank, n, sources):
    handles = fsdp_handles(hf, n, lambda name, off, loc: HostBuffer(
        region(sources[name], off, loc).contiguous() if name in sources else None, loc, torch.bfloat16))
    dests, slices, packed = pull_args(vl, tp, rank, lambda name, shape: torch.full(shape, 0x5A, dtype=torch.uint8))
    return handles, dests, slices, packed, DirectWeightSyncDest()._build_plan(handles, dests, slices, packed=packed)


@pytest.mark.parametrize("rank", range(8))
def test_llama3_8b_tp8_ops_match_the_oracle(rank):
    """Full-size Llama-3-8B (one layer plus embeddings), HF FSDP(8) Shard(0) handles -> vLLM TP8: the ops of every
    fused parameter move exactly what the element rule says, byte for byte; every other name is planned as before."""
    hf = workloads.hf_llama_layout(workloads.LLAMA3_8B, n_layers=1)
    vl = workloads.vllm_tp_layout(hf, workloads.LLAMA3_8B, 8, rank)
    fused_sources = [p.source for _, parts, _ in vl.values() if parts for p in parts]
    sources = host_sources(hf, fused_sources, torch.uint8, rank)
    handles, dests, slices, packed, ops = plan_layout(hf, vl, 8, rank, 8, sources)
    assert set(packed) == {"model.layers.0.self_attn.qkv_proj.weight", "model.layers.0.mlp.gate_up_proj.weight"}
    apply_ops([op for op in ops if op.name in packed], dests)
    np_sources = {n: t.numpy() for n, t in sources.items()}
    for name in packed:
        want = po.destination(vl[name], np_sources, name, fill_value=0x5A)
        assert np.array_equal(dests[name].numpy(), want), name
    # the unpacked names keep the plan they had without packed=
    plain = DirectWeightSyncDest()._build_plan(handles, {n: d for n, d in dests.items() if n not in packed}, slices)
    key = [(op.name, op.src_slices, op.dest_slices, op.rdma_buffer) for op in ops if op.name not in packed]
    assert key == [(op.name, op.src_slices, op.dest_slices, op.rdma_buffer) for op in plain]
    # and the fused names are planned as the unfused pull of the same bytes: one op per (part, shard) it meets
    udests, uslices, _ = unfused_args(vl, hf, 8, rank, lambda name, shape: torch.empty(shape, dtype=torch.uint8))
    uops = DirectWeightSyncDest()._build_plan(handles, udests, uslices)
    assert len(uops) == len(ops)
    assert sorted(map(moved, ops)) == sorted(map(moved, uops))


def moved(op) -> tuple:
    """The (source buffer, source box) an op reads."""
    if op.src_slices is None:
        return id(op.rdma_buffer), tuple((0, e) for e in op.rdma_buffer.shape)
    return id(op.rdma_buffer), tuple((s.start, s.stop) for s in op.src_slices)


LLAMA_SMALL = dict(workloads.LLAMA3_8B, n_layers=2)


@pytest.mark.parametrize("tp,n", [(1, 1), (2, 4), (8, 8), (8, 3)])
def test_scaled_llama_every_rank_matches_the_oracle(tp, n):
    """A scaled-down Llama-3-8B (dim 256, two layers, embeddings) at every rank, FSDP(n) -> vLLM TP(tp), bf16."""
    hf = workloads.hf_llama_layout(workloads.LLAMA3_8B, n_layers=2, scale=16)
    sources = host_sources(hf, list(hf), torch.bfloat16, tp * 10 + n)
    np_sources = {k: v.view(torch.int16).numpy() for k, v in sources.items()}
    for rank in range(tp):
        vl = workloads.vllm_tp_layout(hf, workloads.LLAMA3_8B, tp, rank)
        handles, dests, slices, packed, ops = plan_layout(hf, vl, tp, rank, n, sources)
        dests = {k: torch.full(tuple(vl[k][0]), -3, dtype=torch.int16).view(torch.bfloat16) for k in dests}
        for op in ops:
            op.dest_local = dests[op.name]
        apply_ops(ops, dests)
        for name, entry in vl.items():
            want = po.destination(entry, np_sources, name, fill_value=-3, dtype=np.int16)
            assert np.array_equal(dests[name].view(torch.int16).numpy(), want), (rank, name)


def test_kv_heads_replicated_beyond_tp_read_the_same_rows():
    """A 4-kv-head model at TP8: ranks 2r and 2r + 1 read kv head r, the same source rows."""
    hf = workloads.qwen3_moe_layout(workloads.QWEN3_MOE, n_layers=1, scale=16, n_experts=2, with_embeddings=False)
    starts = []
    for rank in range(8):
        vl = workloads.vllm_tp_layout(hf, workloads.QWEN3_MOE, 8, rank)
        q, k, v = vl["model.layers.0.self_attn.qkv_proj.weight"][1]
        starts.append((k.source_offsets, v.source_offsets))
        assert k.dest_index[0].stop - k.dest_index[0].start == 8  # head_dim 128 / 16
    assert starts[0] == starts[1] != starts[2] == starts[3]


# -- the compiled copy plan, replayed -------------------------------------------------------------------------------
@pytest.mark.parametrize("rank", [0, 5])
def test_compiled_copy_plan_replays_to_the_oracle(rank, monkeypatch):
    """The packed ops' windows through the native plan compiler, replayed on host memory by the C oracle's
    interpreter, write what the numpy oracle says: MoE stacks (an int index dropping the expert dim) included."""
    monkeypatch.setenv("TSB_LINK", "1")
    hf = workloads.qwen3_moe_layout(workloads.QWEN3_MOE, n_layers=1, scale=16, n_experts=4, with_embeddings=False)
    sources = host_sources(hf, list(hf), torch.bfloat16, 7 + rank)
    np_sources = {k: v.view(torch.int16).numpy() for k, v in sources.items()}
    vl = workloads.vllm_tp_layout(hf, workloads.QWEN3_MOE, 8, rank)
    handles, _, slices, packed, _ = plan_layout(hf, vl, 8, rank, 4, sources)
    dests = {k: torch.full(tuple(e[0]), 11, dtype=torch.int16).view(torch.bfloat16) for k, e in vl.items()}
    ops = DirectWeightSyncDest()._build_plan(handles, dests, slices, packed=packed)
    pairs = [DirectWeightSyncDest.op_windows(op, StridedMem.from_tensor(op.rdma_buffer.shard)) for op in ops]
    rects, n = build_rects(pairs)
    table, tiles, info = _native.plan_compile_host(0, rects, n, 0, 256)
    c_oracle.replay_plan(table, tiles, info.tile_bytes // 16, nan_mode=0)
    assert set(packed) >= {"model.layers.0.mlp.experts.w13_weight", "model.layers.0.mlp.experts.w2_weight"}
    for name, entry in vl.items():
        want = po.destination(entry, np_sources, name, fill_value=11, dtype=np.int16)
        assert np.array_equal(dests[name].view(torch.int16).numpy(), want), name


# -- verbatim scale mapping -----------------------------------------------------------------------------------------
class ScaledHost(HostBuffer):
    def __init__(self, shard, scale, granularity, r0, c0):
        super().__init__(shard, shard.shape, E4M3)
        self.scale, self.granularity, self.row0, self.col0 = scale, granularity, r0, c0


def scaled_sources(g, shapes: dict, n, seed):
    """Per source name: FSDP(n) row-shard handles with random fp8 bytes and their own shard-local scales."""
    rng = np.random.default_rng(seed)
    out, full = {}, {}
    for name, shape in shapes.items():
        full[name] = torch.from_numpy(rng.integers(0, 256, size=shape, dtype=np.uint8)).view(E4M3)

        def make(_, off, loc, name=name):
            shard = region(full[name], off, loc).contiguous()
            scale = torch.from_numpy(rng.standard_normal(source_scale_shapes(g, loc, off[-2], off[-1])[0]).astype(np.float32))
            return ScaledHost(shard, scale, g, off[-2], off[-1])
        out.update(fsdp_handles({name: (shape, None)}, n, make))
    return out, full


def scale_at(h, g, idx):
    """The scale of handle ``h`` (source global index ``idx``) as the oracle reads it: the group holding idx."""
    buf = h.rdma_buffer
    grid = buf.scale.reshape(scale_grid(g, buf.shape, buf.row0, buf.col0))
    loc = [i - o for i, o in zip(idx, h.tensor_slice.offsets)]
    lead = tuple(loc[:-2])
    if g == "block":
        return grid[lead + (idx[-2] // 128 - buf.row0 // 128, idx[-1] // 128 - buf.col0 // 128)]
    if g == "channel":
        return grid[lead + (loc[-2], 0)]
    return grid[lead + (0, 0)]


def verbatim_case(g, dest_shape, packed, handles):
    dest = torch.zeros(dest_shape, dtype=torch.uint8).view(E4M3)
    dest_scale = torch.full(source_scale_shapes(g, dest_shape, 0, 0)[0], -7.0)
    ops = DirectWeightSyncDest()._build_plan(handles, {"w": dest}, packed=packed)
    scaled = {"w": (f"{g}_scales", dest, dest_scale, "verbatim")}
    return ops, dest, dest_scale, scaled


@pytest.mark.parametrize("g", ["block", "channel"])
def test_verbatim_packed_groups_that_line_up(g):
    """Fused [q; k; v] with 256/128/128-row parts and a 2-expert stack: each destination group takes the scale of
    the source group holding it (block: the source's global 128-blocks, channel: the source's rows)."""
    handles, full = scaled_sources(g, {"q": (512, 384), "k": (256, 384), "v": (256, 384)}, 2, 3)
    packed = {"w": (PackedPart("q", (slice(0, 256), slice(0, 384)), (256, 0)),
                    PackedPart("k", (slice(256, 384), slice(0, 384)), (128, 0)),
                    PackedPart("v", (slice(384, 512), slice(0, 384)), (0, 0)))}
    ops, dest, dest_scale, scaled = verbatim_case(g, (512, 384), packed, handles)
    rects = DirectWeightSyncDest._verbatim_rects(ops, scaled)["w"]
    grid = dest_scale.reshape(scale_grid(g, (512, 384), 0, 0))
    hits = torch.zeros(grid.shape, dtype=torch.int64)
    for op, src_idx, dst_idx in rects:
        buf = op.rdma_buffer
        grid[dst_idx] = buf.scale.reshape(scale_grid(g, buf.shape, buf.row0, buf.col0))[src_idx]
        hits[dst_idx] += 1
    assert (hits == 1).all()
    step = 128 if g == "block" else 1
    for p in packed["w"]:
        r0, r1 = p.dest_index[0].start, p.dest_index[0].stop
        for r in range(r0, r1, step):
            for c in range(0, 384, 128 if g == "block" else 384):
                src = (p.source_offsets[0] + r - r0, c)
                h = next(h for h in handles[p.source] if h.tensor_slice.offsets[0] <= src[0] <
                         h.tensor_slice.offsets[0] + h.tensor_slice.local_shape[0])
                want = scale_at(h, g, src)
                got = grid[(r // step, c // 128 if g == "block" else 0)]
                assert got.view(torch.int32) == want.view(torch.int32), (p.source, r, c)


def test_verbatim_packed_expert_stack_lines_up():
    g = "block"
    handles, _ = scaled_sources(g, {"e0": (256, 128), "e1": (256, 128)}, 1, 4)
    packed = {"w": tuple(PackedPart(f"e{e}", (e, slice(0, 256), slice(0, 128)), (0, 0)) for e in range(2))}
    ops, dest, dest_scale, scaled = verbatim_case(g, (2, 256, 128), packed, handles)
    rects = DirectWeightSyncDest._verbatim_rects(ops, scaled)["w"]
    grid = dest_scale.reshape(scale_grid(g, (2, 256, 128), 0, 0))
    for op, src_idx, dst_idx in rects:
        buf = op.rdma_buffer
        src_grid = buf.scale.reshape(scale_grid(g, buf.shape, 0, 0)).reshape((1,) + scale_grid(g, buf.shape, 0, 0))
        grid[dst_idx] = src_grid[src_idx]
    for e in range(2):
        assert torch.equal(grid[e], handles[f"e{e}"][0].rdma_buffer.scale)


def test_verbatim_packed_block_straddling_two_parts_is_refused():
    """Qwen3-30B-A3B's w13 at TP8: 96-row gate and up halves, so destination block row 0 straddles both parts."""
    g = "block"
    handles, _ = scaled_sources(g, {"gate": (768, 256), "up": (768, 256)}, 1, 5)
    packed = {"w": (PackedPart("gate", (slice(0, 96), slice(0, 256)), (96, 0)),
                    PackedPart("up", (slice(96, 192), slice(0, 256)), (96, 0)))}
    ops, _, _, scaled = verbatim_case(g, (192, 256), packed, handles)
    with pytest.raises(ValueError, match=r"verbatim pull of 'w' \(block_scales\): destination block \(0, 0\) .* does "
                                         "not lie inside one source group of one handle; requantize=True"):
        DirectWeightSyncDest._verbatim_rects(ops, scaled)


def test_verbatim_packed_part_across_source_blocks_is_refused():
    """A part aligned in the destination but reading from source row 64: its destination block straddles two
    source blocks.  Channel groups (rows) line up all the same."""
    handles, _ = scaled_sources("block", {"a": (384, 128)}, 1, 6)
    packed = {"w": (PackedPart("a", (slice(0, 128), slice(0, 128)), (64, 0)),)}
    ops, _, _, scaled = verbatim_case("block", (128, 128), packed, handles)
    with pytest.raises(ValueError, match=r"destination block \(0, 0\)"):
        DirectWeightSyncDest._verbatim_rects(ops, scaled)
    handles, _ = scaled_sources("channel", {"a": (384, 128)}, 1, 6)
    ops, _, _, scaled = verbatim_case("channel", (128, 128), packed, handles)
    assert len(DirectWeightSyncDest._verbatim_rects(ops, scaled)["w"]) == 1

"""Rotary packed parts without a GPU: the validation of ``rotary_head_dim`` before anything is compiled, the field on
the public path and in the plan key, the rotary oracle pinned by hand and by the torch formula, the planned and
compiled copy plans of Llama-3-8B torchtitan FSDP(8) and FSDP(3) -> vLLM TP8 replayed against the oracle, and the
verbatim scale mapping of rotary block and channel parts."""

import asyncio

import numpy as np
import pytest
import torch

import workloads
from oracle import c_oracle
from oracle import rotary_oracle as ro
from tests.helpers import HostBuffer, fsdp_handles, handles_of, pull_args, region
from tests.test_packed_cpu import ScaledHost, host_sources
from torchstore_b200 import _native, state_dict_utils
from torchstore_b200.direct_weight_sync import (DirectWeightSyncDest, PackedPart, _packed_key, scale_grid,
                                                source_scale_shapes)
from torchstore_b200.planner import StridedMem, build_rects

E4M3 = torch.float8_e4m3fn
LLAMA = workloads.LLAMA3_8B


def check(dest_shape, packed, handles, match):
    dests = {"fused": torch.zeros(dest_shape, dtype=torch.bfloat16)}
    with pytest.raises(ValueError, match=match):
        DirectWeightSyncDest._check_packed(handles, dests, packed)
    with pytest.raises(ValueError, match=match):
        asyncio.run(DirectWeightSyncDest().pull(handles, dests, packed=packed))


# -- the oracle ----------------------------------------------------------------------------------------------------
def test_oracle_hand_written_hd4():
    """Two heads of hd = 4: interleaved rows (a0 b0 a1 b1) become half-split (a0 a1 b0 b1)."""
    src = np.arange(8)[:, None] * 10 + np.arange(2)[None, :]
    want = src[[0, 2, 1, 3, 4, 6, 5, 7]]
    assert np.array_equal(ro.half_split(src, 4), want)
    part = PackedPart("s", (slice(1, 5), slice(0, 2)), (4, 0), rotary_head_dim=4)
    out = ro.fill(np.full((6, 2), -1), [part], {"s": src})
    assert np.array_equal(out[1:5], src[[4, 6, 5, 7]]) and (out[0] == -1).all() and (out[5] == -1).all()


@pytest.mark.parametrize("hd,heads,lead", [(4, 3, ()), (128, 2, ()), (64, 4, (2,))])
def test_oracle_matches_the_torch_formula(hd, heads, lead):
    """torchtitan's and HF's conversion: ``w.view(H, hd // 2, 2, K).transpose(1, 2).reshape(H * hd, K)``."""
    w = torch.randn(lead + (heads * hd, 6))
    want = w.view(lead + (heads, hd // 2, 2, 6)).transpose(-3, -2).reshape(lead + (heads * hd, 6))
    assert np.array_equal(ro.half_split(w.numpy(), hd), want.numpy())
    # the element rule row by row: box row h * hd + t * hd / 2 + j reads source row h * hd + 2j + t
    got = ro.half_split(w.numpy(), hd)
    for h in range(heads):
        for t in (0, 1):
            for j in range(hd // 2):
                assert np.array_equal(got[..., h * hd + t * hd // 2 + j, :], w.numpy()[..., h * hd + 2 * j + t, :])


# -- validation ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hd", [0, -2, 3, True, 2.0, "4"])
def test_head_dim_must_be_a_positive_even_int(hd):
    check((8, 4), {"fused": (PackedPart("a", (slice(0, 8), slice(0, 4)), (0, 0), rotary_head_dim=hd),)},
          {"a": handles_of((8, 4))},
          r"packed destination 'fused' part 0 \(source 'a'\): rotary_head_dim must be None or a positive even int")


def test_source_needs_two_dims():
    check((8, 4), {"fused": (PackedPart("a", (slice(0, 8), 0), (0,), rotary_head_dim=4),)}, {"a": handles_of((8,))},
          r"part 0 \(source 'a'\): rotary_head_dim reorders the rows \(dim -2\) of each head, and the source has 1 dim")


def test_extent_must_be_whole_heads():
    check((8, 4), {"fused": (PackedPart("a", (slice(0, 6), slice(0, 4)), (0, 0), rotary_head_dim=4),)},
          {"a": handles_of((8, 4))}, r"part 0 \(source 'a'\): its extent 6 along the source's dim -2 is not a multiple "
                                     "of rotary_head_dim 4")


def test_heads_start_at_source_row_0():
    check((8, 4), {"fused": (PackedPart("a", (slice(0, 4), slice(0, 4)), (2, 0), rotary_head_dim=4),)},
          {"a": handles_of((8, 4))}, r"part 0 \(source 'a'\): source_offsets\[-2\] \(2\) is not a multiple of "
                                     "rotary_head_dim 4")


def test_coverage_errors_still_name_the_source_element():
    hs = handles_of((16, 4), n=2)[:1]
    check((16, 4), {"fused": (PackedPart("a", (slice(0, 16), slice(0, 4)), (0, 0), rotary_head_dim=4),)}, {"a": hs},
          r"no handle covers global element \(8, 0\) of the source")


def test_plan_key_tells_head_dims_apart():
    def key(hd):
        return _packed_key({"w": (PackedPart("a", (slice(0, 8), slice(0, 4)), (0, 0), rotary_head_dim=hd),)})
    assert len({key(None), key(2), key(4), key(8)}) == 4
    assert key(4) == key(4)


def test_field_rides_in_packed_on_get_state_dict():
    """``get_state_dict(direct_rdma=True, packed=...)`` validates the rotary field before anything is compiled, and
    a valid spec reaches the plan builder (which needs a GPU destination past that point)."""
    hs = handles_of((8, 4), n=2)

    class Store:
        async def get(self, key):
            return 2

        async def get_batch(self, keys):
            return {k: {"a": h} for k, h in zip(keys, hs)}

    store = Store()
    dst = {"w": torch.zeros(8, 4, dtype=torch.bfloat16)}
    try:
        bad = {"w": (PackedPart("a", (slice(0, 8), slice(0, 4)), (0, 0), rotary_head_dim=3),)}
        with pytest.raises(ValueError, match=r"packed destination 'w' part 0 \(source 'a'\): rotary_head_dim must be"):
            asyncio.run(state_dict_utils.get_state_dict(store, "k", dst, direct_rdma=True, packed=bad))
        good = {"w": (PackedPart("a", (slice(0, 8), slice(0, 4)), (0, 0), rotary_head_dim=4),)}
        with pytest.raises(RuntimeError, match="direct weight sync writes GPU memory"):
            asyncio.run(state_dict_utils.get_state_dict(store, "k", dst, direct_rdma=True, packed=good))
    finally:
        state_dict_utils.reset_direct_cache(store)


# -- Llama-3-8B torchtitan -> vLLM TP8 -------------------------------------------------------------------------------
def titan_plan(rank, n, sources, layout):
    vl = workloads.vllm_tp_layout(layout, LLAMA, 8, rank, source="torchtitan")
    handles = fsdp_handles(layout, n, lambda name, off, loc: HostBuffer(
        region(sources[name], off, loc).contiguous() if name in sources else None, loc, sources[name].dtype
        if name in sources else torch.uint8))
    dests, slices, packed = pull_args(vl, 8, rank, lambda name, shape: torch.full(shape, 0x5A, dtype=torch.uint8))
    assert not slices and set(packed) == set(vl)
    return vl, handles, dests, packed


@pytest.mark.parametrize("n", [8, 3])
def test_llama3_8b_torchtitan_tp8_every_rank_matches_the_oracle(n):
    """Full-size Llama-3-8B (one layer, no embeddings), torchtitan FSDP(n) handles -> vLLM TP8 at every rank: the
    planned ops applied on host memory, and the compiled copy plan replayed by the C oracle, both write what
    rotary_oracle says.  FSDP(3)'s uneven shards cut through heads of wq and wk."""
    layout = workloads.llama_layout(LLAMA, n_layers=1, with_embeddings=False)
    cut = 0
    for rank in range(8):
        sources = host_sources(layout, [k for k in layout if "attention.w" in k and "wo" not in k], torch.uint8, rank)
        vl, handles, dests, packed = titan_plan(rank, n, sources, layout)
        name = "model.layers.0.self_attn.qkv_proj.weight"
        q, k, _ = packed[name]
        assert q.rotary_head_dim == k.rotary_head_dim == 128
        ops = [op for op in DirectWeightSyncDest()._build_plan(handles, dests, packed={name: packed[name]})]
        cut += sum(op.rotary is not None and op.rotary[3] == 1 for op in ops)
        np_sources = {s: t.numpy() for s, t in sources.items()}
        want = ro.destination(vl[name], np_sources, name, fill_value=0x5A)
        apply_rotary_ops(ops, dests)
        assert np.array_equal(dests[name].numpy(), want), rank
        # the compiled copy plan, replayed
        dests[name].fill_(0x5A)
        pairs = [DirectWeightSyncDest.op_windows(op, StridedMem.from_tensor(op.rdma_buffer.shard)) for op in ops]
        rects, nr = build_rects(pairs)
        table, tiles, info = _native.plan_compile_host(0, rects, nr, 0, 256)
        c_oracle.replay_plan(table, tiles, info.tile_bytes // 16, nan_mode=0)
        assert np.array_equal(dests[name].numpy(), want), rank
        if n == 8:  # shards of whole heads: one rect per (part, handle), as the HF-named packed pull
            assert len([op for op in ops if op.rotary]) == 2 and nr == 3
    assert (cut > 0) == (n == 3), "FSDP(3)'s shard edges cut heads into head-half pieces"


def apply_rotary_ops(ops, dests):
    """Move every op as its windows say (host tensors, torch strided views)."""
    for op in ops:
        src, dst = DirectWeightSyncDest.op_windows(op, StridedMem.from_tensor(op.rdma_buffer.shard))
        s, d = (torch.as_strided(t, w.shape, w.stride, (w.ptr - t.untyped_storage().data_ptr()) // t.element_size())
                for t, w in ((op.rdma_buffer.shard, src), (dests[op.name], dst)))
        d.copy_(s)


def test_scaled_llama_every_rank_every_name_matches_the_oracle():
    """A scaled-down Llama-3 (dim 256, hd 8, two layers with embeddings), torchtitan FSDP(3) -> vLLM TP2, bf16: every
    vLLM parameter, renamed or fused, holds what rotary_oracle says."""
    layout = workloads.llama_layout(LLAMA, n_layers=2, scale=16)
    sources = host_sources(layout, list(layout), torch.bfloat16, 9)
    np_sources = {k: v.view(torch.int16).numpy() for k, v in sources.items()}
    for rank in range(2):
        vl = workloads.vllm_tp_layout(layout, LLAMA, 2, rank, source="torchtitan")
        handles = fsdp_handles(layout, 3, lambda name, off, loc: HostBuffer(region(sources[name], off, loc).contiguous(),
                                                                            loc, torch.bfloat16))
        dests = {k: torch.full(e[0], -3, dtype=torch.int16).view(torch.bfloat16) for k, e in vl.items()}
        packed = {k: e[1] for k, e in vl.items()}
        ops = DirectWeightSyncDest()._build_plan(handles, dests, packed=packed)
        apply_rotary_ops(ops, dests)
        for name, entry in vl.items():
            want = ro.destination(entry, np_sources, name, fill_value=-3, dtype=np.int16)
            assert np.array_equal(dests[name].view(torch.int16).numpy(), want), (rank, name)


# -- verbatim scale mapping ----------------------------------------------------------------------------------------
def rotary_scaled(g, hd, rows, n):
    rng = np.random.default_rng(hd + n)
    full = torch.from_numpy(rng.integers(0, 256, size=(rows, 256), dtype=np.uint8)).view(E4M3)

    def make(_, off, loc):
        scale = torch.from_numpy(rng.standard_normal(source_scale_shapes(g, loc, off[-2], off[-1])[0]).astype(np.float32))
        return ScaledHost(region(full, off, loc).contiguous(), scale, g, off[-2], off[-1])
    return fsdp_handles({"q": ((rows, 256), None)}, n, make)


def verbatim(g, handles, packed, shape):
    dest = torch.zeros(shape, dtype=torch.uint8).view(E4M3)
    dest_scale = torch.full(source_scale_shapes(g, shape, 0, 0)[0], -7.0)
    ops = DirectWeightSyncDest()._build_plan(handles, {"w": dest}, packed=packed)
    return ops, DirectWeightSyncDest._verbatim_rects(ops, {"w": (f"{g}_scales", dest, dest_scale, "verbatim")})


@pytest.mark.parametrize("g,hd", [("block", 128), ("block", 64), ("channel", 128), ("channel", 8)])
def test_verbatim_rotary_scales_match_a_group_by_group_oracle(g, hd):
    """Each destination group takes the scale of the source group holding the source rows its rows read."""
    handles = rotary_scaled(g, hd, 1024, 2)
    packed = {"w": (PackedPart("q", (slice(0, 512), slice(0, 256)), (256, 0), rotary_head_dim=hd),)}
    _, rects = verbatim(g, handles, packed, (512, 256))
    grid = torch.full(scale_grid(g, (512, 256), 0, 0), -7.0)
    hits = torch.zeros(grid.shape, dtype=torch.int64)
    for op, src_idx, dst_idx in rects["w"]:
        buf = op.rdma_buffer
        src = buf.scale.reshape(scale_grid(g, buf.shape, buf.row0, buf.col0))
        grid[dst_idx] = src[src_idx]
        hits[dst_idx] += 1
    assert (hits == 1).all()
    step = 128 if g == "block" else 1
    for r in range(0, 512, step):
        h, i = divmod(r, hd)
        t, j = divmod(i, hd // 2)
        srow = 256 + h * hd + 2 * j + t
        hh = handles["q"][srow // 512]
        buf = hh.rdma_buffer
        sgrid = buf.scale.reshape(scale_grid(g, buf.shape, buf.row0, buf.col0))
        for c in range(0, 256, 128 if g == "block" else 256):
            want = sgrid[(srow // 128 - buf.row0 // 128, c // 128)] if g == "block" else sgrid[(srow - buf.row0, 0)]
            got = grid[(r // 128, c // 128)] if g == "block" else grid[(r, 0)]
            assert got.view(torch.int32) == want.view(torch.int32), (r, c)


def test_verbatim_rotary_hd256_block_is_refused_naming_the_group():
    """With hd = 256 a 128-row destination block reads the even (or odd) rows of a whole head: two source blocks."""
    handles = rotary_scaled("block", 256, 512, 1)
    packed = {"w": (PackedPart("q", (slice(0, 512), slice(0, 256)), (0, 0), rotary_head_dim=256),)}
    with pytest.raises(ValueError, match=r"verbatim pull of 'w' \(block_scales\): destination block \(0, 0\) .* does "
                                         "not lie inside one source group of one handle"):
        verbatim("block", handles, packed, (512, 256))
    # channel scales move with their rows whatever the head dim
    handles = rotary_scaled("channel", 256, 512, 1)
    verbatim("channel", handles, packed, (512, 256))

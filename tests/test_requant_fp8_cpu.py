"""Requantising pulls without a GPU: the numpy composition oracle pinned to torch CPU's fixture, the native
plan compiler (tsb_requant_fp8_compile_host) replayed on host memory against the oracle for every
(source, destination) granularity pair on FSDP -> TP reshards with unaligned offsets, MoE stacks, ragged
edges and replicated sources, the compiler's errors, and the validation of pull(requantize=True)."""

import asyncio
import os
import time
import types

import numpy as np
import pytest
import torch

from oracle.dequant_fp8_oracle import GRANULARITIES, scale_shape
from oracle.requant_fp8_oracle import (PAIRS, canonical_nan, digest, fixture_inputs, quantize, replay, requantize,
                                       torch_requantize)
from tests.helpers import (Boom, cuda_like, dest_scale_shape, expect_invalid, no_compile, plan_windows, region,
                           shard_box, shard_handles)
from torchstore_b200 import _native
from torchstore_b200.direct_weight_sync import BLOCK, DirectWeightSyncDest, RDMAWeightHandle
from torchstore_b200.planner import StridedMem, build_rects
from torchstore_b200.transport.types import TensorSlice

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "requant_fp8_vectors.npz")
E4M3 = torch.float8_e4m3fn
CODE = {"block": _native.TSB_SCALE_PER_BLOCK, "channel": _native.TSB_SCALE_PER_CHANNEL,
        "tensor": _native.TSB_SCALE_PER_TENSOR}


def same_scale(got: np.ndarray, want: np.ndarray) -> bool:
    got, want = np.asarray(got, np.float32).reshape(-1), np.asarray(want, np.float32).reshape(-1)
    nan = np.isnan(want)
    return np.array_equal(np.isnan(got), nan) and np.array_equal(got[~nan].view(np.uint32), want[~nan].view(np.uint32))


# ---- the oracle against the torch CPU fixture ------------------------------------------------------
def test_fixture_inputs_are_the_recorded_ones():
    d = np.load(GOLDEN)
    inputs = fixture_inputs()
    assert [n for n, *_ in inputs] == list(map(str, d["names"]))
    assert {(sg, dg) for _, sg, dg, *_ in inputs} == set(PAIRS)
    for i, (name, sg, dg, r0, c0, q, s) in enumerate(inputs):
        assert list(map(str, d[f"g{i}"])) == [sg, dg] and list(d[f"off{i}"]) == [r0, c0], name
        assert digest(q.view(torch.uint8).numpy()) == str(d[f"q_sha{i}"]), name
        assert digest(s.numpy().view(np.uint32)) == str(d[f"s_sha{i}"]), name


@pytest.mark.parametrize("i", range(len(fixture_inputs())))
def test_oracle_matches_the_torch_cpu_fixture(i):
    d = np.load(GOLDEN)
    name, sg, dg, r0, c0, q, s = fixture_inputs()[i]
    y, y_scale = requantize(q.view(torch.uint8).numpy(), s.numpy(), sg, r0, c0, dg)
    assert digest(canonical_nan(y)) == str(d[f"y_sha{i}"]), name
    assert same_scale(y_scale, d[f"y_scale{i}"]), name
    ty, ts = torch_requantize(q, s, sg, r0, c0, dg)  # the torch rendering agrees with the numpy composition
    assert np.array_equal(canonical_nan(ty.view(torch.uint8).numpy()), canonical_nan(y)) and same_scale(ts.numpy(), y_scale)


def test_poisoned_scales_poison_their_destination_groups():
    for name, sg, dg, r0, c0, q, s in fixture_inputs():
        if not name.startswith("poison"):
            continue
        _, y_scale = requantize(q.view(torch.uint8).numpy(), s.numpy(), sg, r0, c0, dg)
        assert np.isnan(y_scale).any() and (dg == "tensor" or not np.isnan(y_scale).all()), name


# ---- the plan compiler, replayed on host memory ----------------------------------------------------
def global_scale(g, shape, seed):
    gen = torch.Generator().manual_seed(seed)
    return torch.rand(scale_shape(g, shape), generator=gen) * 0.01 + 1e-4


def local_scale(full_scale, g, off, loc):
    *lead_off, r0, c0 = off
    *lead, n, k = loc
    lead_idx = tuple(slice(o, o + e) for o, e in zip(lead_off, lead))
    if g == "block":
        return full_scale[lead_idx + (slice(r0 // BLOCK, -(-(r0 + n) // BLOCK)), slice(c0 // BLOCK, -(-(c0 + k) // BLOCK)))].contiguous()
    if g == "channel":
        return full_scale[lead_idx + (slice(r0, r0 + n),)].contiguous().reshape(*lead, n, 1)
    return full_scale[lead_idx].contiguous()


class FakeScaledBuffer:
    """Host-memory stand-in for ScaledNvlinkBuffer (the planner only reads these attributes)."""

    def __init__(self, shard, scale, g, r0, c0):
        self.shard, self.scale, self.granularity, self.row0, self.col0 = shard, scale, g, r0, c0
        self.dtype = shard.dtype


def compile_pull(q_full, full_scale, sg, src_boxes, dst_box, dg, flags=0):
    """Plan a requantising pull of `q_full`'s `sg`-scaled shards into a `dg`-scaled fp8 window `dst_box` with the
    plan `flags`; returns (dest, dest_scale, tables, keepalive)."""
    handles, keep = shard_handles(q_full, src_boxes, lambda shard, off, loc: FakeScaledBuffer(
        shard, local_scale(full_scale, sg, off, loc), sg, off[-2], off[-1]))
    loc = dst_box[1]
    dest = torch.full(loc, 0x55, dtype=torch.uint8).view(E4M3)
    dest_scale = torch.full(dest_scale_shape(dg, loc), -1.0)
    ops, pairs = plan_windows(handles, dest, dst_box)
    sources, index = [], {}
    for op in ops:
        buf = op.rdma_buffer
        if id(buf) not in index:
            index[id(buf)] = len(sources)
            n, k = buf.shard.shape[-2:]
            sources.append(_native.DqSource(buf.shard.data_ptr(), buf.scale.data_ptr(), buf.shard.numel() // (n * k), n, k,
                                            buf.row0, buf.col0, CODE[sg], 0))
    rects, nr = build_rects(pairs)
    for i in range(nr):
        rects[i].src_dtype = rects[i].dst_dtype = _native.TSB_F8E4M3
    arr = _native.make_dq_source_array(max(1, len(sources)))
    for i, s in enumerate(sources):
        arr[i] = s
    n, k = loc[-2:]
    tgt = _native.make_sq_target_array(1)
    tgt[0] = _native.SqTarget(dest.data_ptr(), dest_scale.data_ptr(), dest.numel() // (n * k), n, k, CODE[dg], 0)
    tables = _native.requant_fp8_compile_host(0, rects, nr, arr, len(sources), tgt, 1, flags)
    return dest, dest_scale, tables, (keep, rects, arr, tgt, handles)


def run_reshard(q_full, full_scale, sg, src_boxes, dst_box, dg):
    dest, dest_scale, tables, _keep = compile_pull(q_full, full_scale, sg, src_boxes, dst_box, dg)
    replay(*tables)
    want_q, want_s = requantize(region(q_full, *dst_box).view(torch.uint8).numpy(),
                                local_scale(full_scale, sg, *dst_box).numpy(), sg, dst_box[0][-2], dst_box[0][-1], dg)
    assert np.array_equal(dest.view(torch.uint8).numpy(), want_q)
    assert np.array_equal(dest_scale.numpy().reshape(-1).view(np.uint32), np.asarray(want_s, np.float32).reshape(-1).view(np.uint32))
    return tables


def fp8_full(shape, seed):
    gen = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=gen) * 4).to(E4M3)


@pytest.mark.parametrize("sg,dg", PAIRS)
@pytest.mark.parametrize("n,dst_dim", [(6, 0), (6, 1), (4, 0)])
def test_fsdp_rows_to_tp_reshard_replays_to_the_oracle(sg, dg, n, dst_dim):
    """FSDP(n) row shards starting mid-block (300 rows over 6: 50-row shards) into row-parallel (rows 0..150,
    150..300) and column-parallel (columns 0..130, 130..260) TP destinations, neither 128-aligned."""
    q = fp8_full((300, 260), 10 * n + dst_dim)
    s = global_scale(sg, q.shape, n)
    srcs = [shard_box(q.shape, n, r, 0) for r in range(n)]
    for d in range(2):
        run_reshard(q, s, sg, srcs, shard_box(q.shape, 2, d, dst_dim), dg)


@pytest.mark.parametrize("sg,dg", PAIRS)
def test_moe_stack_and_ragged_edges(sg, dg):
    q = fp8_full((4, 130, 260), 5)
    s = global_scale(sg, q.shape, 5)
    experts = [shard_box(q.shape, 2, r, 0) for r in range(2)]  # EP: experts 0-1 and 2-3
    run_reshard(q, s, sg, experts, ((0, 0, 0), (4, 130, 260)), dg)
    rows = [shard_box(q.shape, 3, r, 1) for r in range(3)]  # rows cut at 44 / 88, mid-block
    for d in range(2):
        run_reshard(q, s, sg, rows, shard_box(q.shape, 2, d, 2), dg)
    q = fp8_full((203, 77), 6)  # ragged: nothing is a multiple of 16
    s = global_scale(sg, q.shape, 6)
    run_reshard(q, s, sg, [shard_box(q.shape, 3, r, 1) for r in range(3)], ((0, 0), (203, 77)), dg)


@pytest.mark.parametrize("sg,dg", PAIRS)
def test_replicated_sources_are_read_once(sg, dg):
    q = fp8_full((256, 200), 4)
    s = global_scale(sg, q.shape, 4)
    srcs = [shard_box(q.shape, 2, r % 2, 0) for r in range(4)]  # (Replicate, Shard(0)): every shard twice
    units, pieces, tiles, _ = run_reshard(q, s, sg, srcs, ((0, 0), (256, 200)), dg)
    read = int((pieces["rows"].astype(np.int64) * pieces["cols"]).sum()) + int((tiles["rows"].astype(np.int64) * tiles["cols"]).sum())
    assert read == 256 * 200


def test_moe_intermediate_96_rows_per_rank():
    """MoE intermediate size 768 over 8 ranks: 96-row destinations whose blocks no source scale describes."""
    q = fp8_full((2, 768, 256), 9)
    s = global_scale("block", q.shape, 9)
    for d in (1, 5):
        units, pieces, _, _ = run_reshard(q, s, "block", [((0, 0, 0), (2, 768, 256))], shard_box(q.shape, 8, d, 1), "block")
        assert (units["rows"] == 96).all() and len(units) == 2 * 2
        assert len(pieces) == 2 * 2 * 2  # each destination block straddles a source block row


@pytest.mark.parametrize("g", GRANULARITIES)
def test_aligned_identity(g):
    """Formula-quantised finite data, same granularity and aligned groups: the fp8 bytes come back unchanged."""
    x = torch.randn(256, 384, generator=torch.Generator().manual_seed(3)) * 3
    q_np, s_np = quantize(x.numpy(), g)
    q = torch.from_numpy(q_np).view(E4M3)
    s = torch.from_numpy(np.asarray(s_np, np.float32).copy()).reshape(scale_shape(g, q.shape))
    dest, dest_scale, tables, keep = compile_pull(q, s, g, [shard_box(q.shape, 2, r, 0) for r in range(2)], ((0, 0), (256, 384)), g)
    replay(*tables)  # writes dest and dest_scale, reads the shards in keep
    assert np.array_equal(dest.view(torch.uint8).numpy(), q_np)


def test_per_channel_kernel_paths():
    """Rows of up to 32 KiB take the staged bands, longer rows the two-pass tiles; per tensor is two-pass."""
    q = fp8_full((4, 40000), 2)
    s = global_scale("block", q.shape, 2)
    units, pieces, tiles, n_groups = run_reshard(q, s, "block", [((0, 0), (4, 40000))], ((0, 0), (4, 40000)), "channel")
    assert len(units) == 0 and n_groups == 4 and (tiles["scale_inv"] != 0).sum() == 4
    units, _, tiles, _ = run_reshard(q[:, :4096].contiguous(), s[:, :32].contiguous(), "block", [((0, 0), (4, 4096))],
                                     ((0, 0), (4, 4096)), "channel")
    assert len(tiles) == 0 and (units["per_row"] == 1).all()


def test_full_size_llama3_8b_compile():
    """Llama-3-8B w1 [14336, 4096] from 6 block-scaled FSDP row shards (boundaries mid-block) into a per-channel
    destination, compiled from addresses alone: no memory behind them is touched."""
    rows, cols, n_src = 14336, 4096, 6
    src_base, dst_base, scale_base = 1 << 40, 1 << 41, 1 << 42
    pairs, sources = [], _native.make_dq_source_array(n_src)
    for r in range(n_src):
        r0, r1 = r * rows // n_src, (r + 1) * rows // n_src
        src = StridedMem(src_base + r * (1 << 30), (r1 - r0, cols), (cols, 1), E4M3, 0)
        dst = StridedMem(dst_base + r0 * cols, (r1 - r0, cols), (cols, 1), E4M3, 0)
        pairs.append((src, dst))
        sources[r] = _native.DqSource(src.ptr, scale_base + r * (1 << 20), 1, r1 - r0, cols, r0, 0, CODE["block"], 0)
    rects, n = build_rects(pairs)
    for i in range(n):
        rects[i].src_dtype = rects[i].dst_dtype = _native.TSB_F8E4M3
    tgt = _native.make_sq_target_array(1)
    tgt[0] = _native.SqTarget(dst_base, scale_base + (1 << 30), 1, rows, cols, CODE["channel"], 0)
    t0 = time.perf_counter()
    units, pieces, tiles, _ = _native.requant_fp8_compile_host(0, rects, n, sources, n_src, tgt, 1)
    assert time.perf_counter() - t0 < 2.0
    assert len(tiles) == 0 and int(units["rows"].astype(np.int64).sum()) == rows
    assert int((pieces["rows"].astype(np.int64) * pieces["cols"]).sum()) == rows * cols
    assert (pieces["vec"] == 1).all()


# ---- compiler errors ------------------------------------------------------------------------------
def test_compile_errors_name_the_target_group_rect_or_source():
    q = torch.zeros(256, 256, dtype=E4M3)
    s = torch.zeros(2, 2)
    dst = torch.zeros(256, 256, dtype=torch.uint8).view(E4M3)
    dscale = torch.zeros(256)

    def compile_with(windows=None, src_kw=(), tgt_kw=()):
        f = dict(src=q.data_ptr(), scale=s.data_ptr(), batch=1, rows=256, cols=256, row0=0, col0=0,
                 granularity=_native.TSB_SCALE_PER_BLOCK, pad=0)
        f.update(src_kw)
        arr = _native.make_dq_source_array(1)
        arr[0] = _native.DqSource(**f)
        t = dict(dst=dst.data_ptr(), scale_inv=dscale.data_ptr(), batch=1, rows=256, cols=256,
                 granularity=_native.TSB_SCALE_PER_CHANNEL, pad=0)
        t.update(tgt_kw)
        tgt = _native.make_sq_target_array(1)
        tgt[0] = _native.SqTarget(**t)
        rects, n = build_rects(windows or [(StridedMem.from_tensor(q), StridedMem.from_tensor(dst))])
        for i in range(n):
            rects[i].src_dtype = rects[i].dst_dtype = _native.TSB_F8E4M3
        return _native.requant_fp8_compile_host(0, rects, n, arr, 1, tgt, 1)

    assert len(compile_with()[0]) == 256 // 128  # bands of 128 rows of 256 bytes
    half = [(StridedMem.from_tensor(q[:100]), StridedMem.from_tensor(dst[:100]))]  # rows 100.. never written
    assert "target 0 group (0, 100)" in expect_invalid(lambda: compile_with(half))
    assert "target 0 group (0, 0, 0)" in expect_invalid(lambda: compile_with(half, tgt_kw=dict(granularity=_native.TSB_SCALE_PER_BLOCK)))
    assert "target 0 group (0)" in expect_invalid(lambda: compile_with(half, tgt_kw=dict(granularity=_native.TSB_SCALE_PER_TENSOR)))
    twice = [(StridedMem.from_tensor(q), StridedMem.from_tensor(dst))] * 2  # every element written twice
    assert "exactly once" in expect_invalid(lambda: compile_with(twice))
    for kw in (dict(granularity=0), dict(granularity=4), dict(pad=1)):
        assert "target 0" in expect_invalid(lambda: compile_with(tgt_kw=kw))
    for kw in (dict(granularity=0), dict(scale=0), dict(pad=1)):
        assert "source 0" in expect_invalid(lambda: compile_with(src_kw=kw))
    assert "rect 0" in expect_invalid(lambda: compile_with(src_kw=dict(src=q.data_ptr() + (1 << 20))))  # in no source
    # a source of 128-byte rows read as 256-byte rows: every rect row crosses a source row
    assert "rect 0" in expect_invalid(lambda: compile_with(src_kw=dict(rows=512, cols=128, scale=s.data_ptr())))


# ---- pull validation (before anything is compiled) --------------------------------------------------
no_compile = pytest.fixture(no_compile)


def handles(kinds, dtype=E4M3):
    return [RDMAWeightHandle(rdma_buffer=types.SimpleNamespace(granularity=k, dtype=dtype), source_rank=r,
                             tensor_slice=TensorSlice((0, 0), (r,), (8, 8), (8, 8), (2,))) for r, k in enumerate(kinds)]


def test_pull_validation(no_compile):
    check = DirectWeightSyncDest._check_scales
    dest = {"w": cuda_like(torch.zeros(8, 8, dtype=E4M3))}
    scales = {"block_scales": {"w": torch.zeros(1, 1)}}
    # the default refusal is unchanged, with a hint
    with pytest.raises(TypeError, match="bf16, f16 or f32 handles.*requantize=True"):
        check({"w": handles(["block"])}, dest, scales)
    assert check({"w": handles(["block", "block"])}, dest, scales, requantize=True)["w"][0] == "block_scales"
    with pytest.raises(ValueError, match="mix scaled fp8 and unscaled"):
        check({"w": handles(["block", None])}, dest, scales, requantize=True)
    with pytest.raises(ValueError, match="granularities"):
        check({"w": handles(["block", "tensor"])}, dest, {"channel_scales": {"w": torch.zeros(8, 1)}}, requantize=True)
    with pytest.raises(TypeError, match="bf16, f16 or f32 handles"):  # unscaled fp8 handles have nothing to requantise from
        check({"w": handles([None])}, dest, {"tensor_scales": {"w": torch.zeros(())}}, requantize=True)
    # bf16 handles into a scaled destination still quantise with the flag
    assert check({"w": handles([None], torch.bfloat16)}, dest, scales, requantize=True)["w"][0] == "block_scales"
    # through pull(): raised before any plan is compiled
    with pytest.raises(ValueError, match="mix"):
        asyncio.run(DirectWeightSyncDest().pull({"w": handles(["block", None])}, dest, block_scales=scales["block_scales"],
                                                requantize=True))
    with pytest.raises(TypeError, match="bf16, f16 or f32 handles"):
        asyncio.run(DirectWeightSyncDest().pull({"w": handles(["block"])}, dest, block_scales=scales["block_scales"]))


def test_plan_cache_key_includes_the_flag():
    """A cached plan built without requantize=True is dropped when the flag is set, and vice versa."""
    for built, flag in ((False, True), (True, False)):
        d = DirectWeightSyncDest()
        d._plan = []
        d._plan_key = (frozenset({("w", "block_scales")}), built, None)
        d.close = lambda: (_ for _ in ()).throw(Boom("rebuilt"))
        with pytest.raises(Boom):
            asyncio.run(d.pull({}, {}, block_scales={"w": torch.zeros(1, 1)}, requantize=flag))


def test_store_path_refuses_the_flag():
    from torchstore_b200 import state_dict_utils

    with pytest.raises(NotImplementedError, match="requantize"):
        asyncio.run(state_dict_utils.get_state_dict(None, "k", {"w": torch.zeros(1)}, direct_rdma=False, requantize=True))

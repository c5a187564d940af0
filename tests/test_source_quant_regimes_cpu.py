"""The source-side quantisation catalogue (tests/source_quant_regimes.py) without a GPU: every named workload
compiled on host memory, its tables replayed with the oracle interpreter and compared with ``quantize``, and
every regime shown to hold on its workload's tables.  Then the consumers of source-quantised handles, whose
shards carry *different* scales for the groups they share: the dequantising and requantising pull plans over
such shards, compiled through the planner path of a direct pull and replayed against per-shard references."""

import functools

import numpy as np
import pytest
import torch

from oracle import dequant_fp8_oracle, requant_fp8_oracle
from oracle.source_quant_oracle import GRANULARITIES, bits_of, element_scales, quantize, replay, synth_f32, widen
from tests.helpers import dest_scale_shape, plan_windows, region, shard_box
from tests.source_quant_regimes import REGIMES, WORKLOADS, plan_bytes
from tests.test_requant_fp8_cpu import CODE, FakeScaledBuffer
from tests.test_source_quant_cpu import compile_host, host_shard
from torchstore_b200 import _native
from torchstore_b200.direct_weight_sync import RDMAWeightHandle
from torchstore_b200.planner import build_rects
from torchstore_b200.transport.types import TensorSlice

E4M3 = torch.float8_e4m3fn

# Every regime the catalogue names.  A regime added there without a workload that reaches it, or dropped
# from it, fails test_catalogue_is_complete until this list says so too.
EXPECTED = [
    "block_unit_vec_bfloat16", "block_unit_vec_float16", "block_unit_vec_float32",
    "block_unit_bytewise_bfloat16", "block_unit_bytewise_float16", "block_unit_bytewise_float32",
    "block_partial_first_and_last",
    "band_lane_atomics", "band_warp_reduced", "band_mixed_fold", "band_256_rows", "band_256_rows_f32",
    "band_1024_chunks", "band_crosses_matrix", "band_bytewise",
    "band_one_row_at_stage_bound_bfloat16", "band_one_row_at_stage_bound_float16", "band_one_row_at_stage_bound_float32",
    "two_pass_first_width_past_stage_bf16", "two_pass_first_width_past_stage_f32",
    "tensor_tiles_with_remainder", "two_pass_over_256_groups_tensor", "two_pass_over_256_groups_channel",
    "two_pass_bytewise_bfloat16", "two_pass_bytewise_float16", "two_pass_bytewise_float32",
    "three_dtype_launches", "units_and_tiles",
]


def test_catalogue_is_complete():
    assert sorted(REGIMES) == sorted(EXPECTED)
    assert {r.workload for r in REGIMES.values()} == set(WORKLOADS)  # every regime has a workload and vice versa


def workload_inputs(name):
    """One synthetic shard per target of workload `name`, in its dtype."""
    w = WORKLOADS[name]
    return [synth_f32(t.shape, w.seed + 7 * i).to(getattr(torch, t.dtype)) for i, t in enumerate(w.targets)]


@functools.lru_cache(maxsize=None)
def replayed(name):
    """Compile workload `name` on host memory, replay its tables, check every target against the oracle and
    return (tables, targets).  The addresses are stale afterwards: predicates only compare them."""
    w = WORKLOADS[name]
    keep, targets = [], []
    for t, x in zip(w.targets, workload_inputs(name)):
        backing, q, s, tgt = host_shard(x, t.granularity, t.row0, t.col0, t.misalign)
        keep.append((x, q, s, backing))
        targets.append(tgt)
    tables = compile_host(targets)
    replay(*tables)
    for t, (x, q, s, _) in zip(w.targets, keep):
        want_q, want_s = quantize(widen(bits_of(x), t.dtype), t.granularity, t.row0, t.col0)
        assert np.array_equal(q, want_q), t.describe()
        assert np.array_equal(s.view(np.uint32), want_s.view(np.uint32)), t.describe()
    assert plan_bytes(tables)[1] == sum(x.numel() * x.element_size() for x in workload_inputs(name))
    return tables, [_native.SourceQuantTarget.from_buffer_copy(t) for t in targets]


@pytest.mark.parametrize("name", sorted(WORKLOADS))
def test_workload_replays_to_the_oracle(name):
    replayed(name)


@pytest.mark.parametrize("regime", sorted(REGIMES))
def test_regime_is_hit_by_its_workload(regime):
    r = REGIMES[regime]
    tables, targets = replayed(r.workload)
    assert r.holds(tables, targets), f"{regime} ({r.doc}) not reached by {WORKLOADS[r.workload].describe()}"


# ---------------------------------------------------------------------------------------------
# consumers of shard-local scales
# ---------------------------------------------------------------------------------------------
# global shape and source boxes (offset, local shape): every layout has groups that two shards share
SHARD_LAYOUTS = {
    "cols_at_70": ((300, 260), (((0, 0), (300, 70)), ((0, 70), (300, 190)))),
    "rows_75r_cols_130": ((300, 260), tuple(((75 * r, c), (75, 130)) for r in range(4) for c in (0, 130))),
    "ep_rows_100_cols_130": ((4, 200, 260), tuple(((e, r, c), (2, 100, 130)) for e in (0, 2) for r in (0, 100) for c in (0, 130))),
    "replicas_rows_150_cols_130": ((300, 260), tuple(((r, c), (150, 130)) for r in (0, 150) for c in (0, 130)) * 2),
}
# source dtype of each granularity's shards
SRC_DTYPE = {"block": torch.bfloat16, "channel": torch.float32, "tensor": torch.float16}


def windows(shape):
    """Destination windows of a consumer pull: the whole tensor, its second row half (mid-block), its second
    column half."""
    return {"whole": ((0,) * len(shape), tuple(shape)), "rows": shard_box(shape, 2, 1, len(shape) - 2),
            "cols": shard_box(shape, 2, 1, len(shape) - 1)}


# (consumer, window) of every pull a layout gets: dequantise into each dtype, requantise into each granularity, raw
CONSUMERS = (("bfloat16", "whole"), ("float16", "rows"), ("float32", "cols"),
             ("block", "cols"), ("channel", "whole"), ("tensor", "rows"), ("raw", "whole"))


def oracle_shards(x_full, g, boxes):
    """The oracle staging of every source box: [(offset, local shape, fp8 bytes uint8, scale_inv float32)]."""
    out = []
    for off, loc in boxes:
        shard = region(x_full, off, loc).contiguous()
        q, s = quantize(widen(bits_of(shard), str(shard.dtype)[6:]), g, off[-2], off[-1])
        out.append((off, loc, q, np.asarray(s, dtype=np.float32)))
    return out


def group_keys(g, off, loc) -> np.ndarray:
    """The global group of every element of a box, as one integer per element."""
    *lead_off, r0, c0 = off
    *lead, n, k = loc
    m = np.zeros((), dtype=np.int64)
    for o, e in zip(lead_off, lead):
        m = m[..., None] * 1000 + (o + np.arange(e))
    m = m[..., None, None]
    rows, cols = (r0 + np.arange(n))[:, None], (c0 + np.arange(k))[None, :]
    if g == "block":
        key = (m * 1000 + rows // 128) * 1000 + cols // 128
    elif g == "channel":
        key = m * 100000 + rows + 0 * cols
    else:
        key = m + 0 * rows + 0 * cols
    return np.broadcast_to(key, tuple(loc))


def assert_shared_groups_differ(shards, g):
    """Two shards hold different scale_inv values for one global group: otherwise a consumer that reads the
    wrong shard's scale would pass."""
    seen = {}
    for i, (off, loc, _, s) in enumerate(shards):
        keys = group_keys(g, off, loc).reshape(-1)
        vals = np.ascontiguousarray(element_scales(s, g, loc, off[-2], off[-1])).reshape(-1).view(np.uint32)
        uk, first = np.unique(keys, return_index=True)
        for key, v in zip(uk.tolist(), vals[first].tolist()):
            seen.setdefault(key, {})[i] = v
    assert any(len(set(by_shard.values())) > 1 for by_shard in seen.values()), f"no {g} group with two scales"


def assemble(shape, shards, g):
    """Global fp8 bytes and per-element f32 scales of the shards (a replica overwrites its twin's equal values)."""
    q = np.zeros(shape, dtype=np.uint8)
    e = np.zeros(shape, dtype=np.float32)
    for off, loc, sq, ss in shards:
        idx = tuple(slice(o, o + n) for o, n in zip(off, loc))
        q[idx] = sq
        e[idx] = element_scales(ss, g, loc, off[-2], off[-1])
    return q, e


def want_consumer(shape, shards, g, consumer, window):
    """The per-shard reference of one consumer over `window`: raw bytes, dequantised bits (uint16/uint32), or
    requantised (bytes, scale_inv)."""
    q, e = assemble(shape, shards, g)
    idx = tuple(slice(o, o + n) for o, n in zip(*window))
    if consumer == "raw":
        return q[idx]
    with np.errstate(all="ignore"):
        x = (dequant_fp8_oracle.decode_e4m3(q[idx]) * e[idx]).astype(np.float32)
    if consumer in dequant_fp8_oracle.DST:
        return dequant_fp8_oracle.narrow(x, consumer)
    return requant_fp8_oracle.quantize(x, consumer)


def compile_consumer(shape, shards, g, consumer, window):
    """Plan a dequantising (`consumer` a dtype) or requantising (`consumer` a granularity) pull of host shards
    that each carry their own scale, through the planner path of a direct pull -> (dest, dest_scale, tables,
    keepalive)."""
    handles, keep = [], []
    for r, (off, loc, sq, ss) in enumerate(shards):
        shard = torch.from_numpy(np.ascontiguousarray(sq)).view(E4M3)
        scale = torch.from_numpy(np.ascontiguousarray(ss))
        keep += [shard, scale]
        buf = FakeScaledBuffer(shard, scale, g, off[-2], off[-1])
        handles.append(RDMAWeightHandle(rdma_buffer=buf, tensor_slice=TensorSlice(off, (r,), shape, loc, (len(shards),)),
                                        source_rank=r))
    loc = window[1]
    requant = consumer in GRANULARITIES
    dest = torch.full(loc, 0x55, dtype=torch.uint8).view(E4M3) if requant else torch.zeros(loc, dtype=getattr(torch, consumer))
    dest_scale = torch.full(dest_scale_shape(consumer, loc), -1.0) if requant else None
    ops, pairs = plan_windows(handles, dest, window)
    sources, index = [], {}
    for op in ops:
        buf = op.rdma_buffer
        if id(buf) not in index:
            index[id(buf)] = len(sources)
            n, k = buf.shard.shape[-2:]
            sources.append(_native.DqSource(buf.shard.data_ptr(), buf.scale.data_ptr(), buf.shard.numel() // (n * k), n, k,
                                            buf.row0, buf.col0, CODE[g], 0))
    rects, nr = build_rects(pairs)
    arr = _native.make_dq_source_array(max(1, len(sources)))
    for i, s in enumerate(sources):
        arr[i] = s
    if not requant:
        return dest, None, _native.dequant_fp8_compile_host(0, rects, nr, arr, len(sources)), (keep, rects, arr)
    for i in range(nr):
        rects[i].src_dtype = rects[i].dst_dtype = _native.TSB_F8E4M3
    n, k = loc[-2:]
    tgt = _native.make_sq_target_array(1)
    tgt[0] = _native.SqTarget(dest.data_ptr(), dest_scale.data_ptr(), dest.numel() // (n * k), n, k, CODE[consumer], 0)
    tables = _native.requant_fp8_compile_host(0, rects, nr, arr, len(sources), tgt, 1)
    return dest, dest_scale, tables, (keep, rects, arr, tgt)


def layout_shards(layout, g, seed):
    shape, boxes = SHARD_LAYOUTS[layout]
    x = synth_f32(shape, seed).to(SRC_DTYPE[g])
    return shape, boxes, x, oracle_shards(x, g, boxes)


@pytest.mark.parametrize("g", GRANULARITIES)
@pytest.mark.parametrize("layout", sorted(SHARD_LAYOUTS))
def test_consumer_plans_of_shard_local_scales_replay_to_per_shard_references(layout, g):
    shape, _, _, shards = layout_shards(layout, g, 300 + len(layout))
    assert_shared_groups_differ(shards, g)
    for consumer, win in CONSUMERS:
        if consumer == "raw":
            continue
        window = windows(shape)[win]
        dest, dest_scale, tables, _keep = compile_consumer(shape, shards, g, consumer, window)
        want = want_consumer(shape, shards, g, consumer, window)
        where = f"{layout} {g} -> {consumer} over the {win} window"
        if dest_scale is None:
            dequant_fp8_oracle.replay(tables)
            got = dest.view(torch.int16 if dest.element_size() == 2 else torch.int32).numpy().view(want.dtype)
            assert np.array_equal(got, want), where
        else:
            requant_fp8_oracle.replay(*tables)
            assert np.array_equal(dest.view(torch.uint8).numpy(), want[0]), where
            assert np.array_equal(dest_scale.numpy().reshape(-1).view(np.uint32),
                                  np.asarray(want[1], np.float32).reshape(-1).view(np.uint32)), where


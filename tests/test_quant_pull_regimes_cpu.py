"""The quantising-pull catalogue (tests/quant_pull_regimes.py) without a GPU: every named workload planned on
host memory through the planner of a direct pull, its block and per-channel / per-tensor tables replayed
with the oracle interpreters and compared bit for bit with the oracles' quantisation of each destination
window, and every regime shown to hold on its workload's tables."""

import functools

import numpy as np
import pytest
import torch

from oracle import block_fp8_oracle, scaled_fp8_oracle
from tests.helpers import dest_scale_shape, rand_full, region
from tests.quant_pull_regimes import REGIMES, WORKLOADS, compile_tables, plan_bytes, spots
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, RDMAWeightHandle
from torchstore_b200.planner import StridedMem
from torchstore_b200.transport.types import TensorSlice

E4M3 = torch.float8_e4m3fn

# Every regime the catalogue names.  A regime added there without a workload that reaches it, or dropped
# from it, fails test_catalogue_is_complete until this list says so too.
EXPECTED = [
    "block_all_vec_bfloat16", "block_all_vec_float16", "block_all_vec_float32",
    "block_byte_piece_bfloat16", "block_byte_piece_float16", "block_byte_piece_float32",
    "block_vec_and_byte_pieces", "block_of_8_pieces", "block_pitch_off_16", "block_piece_off_16_columns",
    "block_under_16_columns", "block_one_row", "block_partial_corner_in_stack", "block_mixed_dtypes",
    "block_replica_read_once",
    "band_256_rows_bfloat16", "band_256_rows_float32", "band_129_to_255_rows",
    "band_vec_steps_span_rows", "band_vec_steps_in_one_row", "band_vec_steps_mixed",
    "band_byte_steps_span_rows", "band_byte_steps_in_one_row", "band_byte_steps_mixed",
    "band_piece_off_16_columns", "band_padded_stage_pitch",
    "band_one_row_at_stage_bound_bfloat16", "band_one_row_at_stage_bound_float16", "band_one_row_at_stage_bound_float32",
    "band_in_stack", "band_mixed_dtypes",
    "tile_tensor_rows_vec", "tile_tensor_rows_byte", "tile_tensor_group_over_mesh", "tile_channel_rows_over_stage",
    "tile_full_width_and_remainder", "tile_over_256_groups", "bands_and_tiles",
]


def test_catalogue_is_complete():
    assert sorted(REGIMES) == sorted(EXPECTED)
    assert {r.workload for r in REGIMES.values()} == set(WORKLOADS)  # every regime has a workload and vice versa


def workload_inputs(name):
    """The global source tensor of every name of workload `name`, in its dtype."""
    w = WORKLOADS[name]
    return [rand_full(p.shape, getattr(torch, p.dtype), w.seed + 7 * i) for i, p in enumerate(w.pulls)]


def host_shard(x, off, loc, misalign):
    """region(x, off, loc) in a fresh host allocation, starting `misalign` elements past its (aligned) start."""
    n = int(np.prod(loc, dtype=np.int64))
    flat = torch.zeros(n + misalign + 64, dtype=x.dtype)
    out = flat[misalign: misalign + n].view(loc)
    out.copy_(region(x, off, loc))
    return out


def oracle_quantize(x, g):
    """The numpy oracle of granularity `g` over float32 values x -> (fp8 bytes, scale_inv)."""
    return block_fp8_oracle.quantize(x) if g == "block" else scaled_fp8_oracle.quantize(x, g)


@functools.lru_cache(maxsize=None)
def compiled(name, flags=0):
    """Plan workload `name` on host memory with the plan `flags` -> (tables, geometry, xs, dests, scales,
    keepalive).  The destinations are zero; the addresses stay valid while the result is cached."""
    w = WORKLOADS[name]
    xs = workload_inputs(name)
    handles, dests, scales, slices = {}, {}, {}, {}
    for i, (p, x) in enumerate(zip(w.pulls, xs)):
        n = f"w{i}"
        handles[n] = [RDMAWeightHandle(rdma_buffer=host_shard(x, off, loc, p.shift(r)),
                                       tensor_slice=TensorSlice(off, (r,), p.shape, loc, (len(p.src),)), source_rank=r)
                      for r, (off, loc) in enumerate(p.src)]
        off, loc = p.dst
        dests[n] = torch.zeros(loc, dtype=E4M3)
        scales[n] = torch.zeros(dest_scale_shape(p.g, loc), dtype=torch.float32)
        slices[n] = TensorSlice(off, (0,), p.shape, loc, (1,))
    ops = DirectWeightSyncDest()._build_plan(handles, dests, slices)
    tables, geom = compile_tables(w.pulls, ops, handles, StridedMem.from_tensor, dests, scales, flags)
    return tables, geom, xs, dests, scales, handles


@pytest.mark.parametrize("name", sorted(WORKLOADS))
def test_workload_replays_to_the_oracle(name):
    tables, _, xs, dests, scales, handles = compiled(name)
    w = WORKLOADS[name]
    if tables.block is not None:
        block_fp8_oracle.replay(*tables.block)
    if tables.scaled is not None:
        scaled_fp8_oracle.replay(*tables.scaled)
    read = 0
    for i, (p, x) in enumerate(zip(w.pulls, xs)):
        want_q, want_s = oracle_quantize(region(x, *p.dst).float().numpy(), p.g)
        n = f"w{i}"
        assert np.array_equal(dests[n].view(torch.uint8).numpy(), want_q), p.describe()
        assert np.array_equal(scales[n].numpy().reshape(-1).view(np.uint32), np.asarray(want_s, np.float32).reshape(-1).view(np.uint32)), \
            p.describe()
        read += dests[n].numel() * x.element_size()
    assert sum(b for _, b in plan_bytes(tables).values()) == read  # every destination element read once


@pytest.mark.parametrize("regime", sorted(REGIMES))
def test_regime_is_hit_by_its_workload(regime):
    r = REGIMES[regime]
    tables, geom, *_ = compiled(r.workload)
    assert r.holds(tables, geom), f"{regime} ({r.doc}) not reached by {WORKLOADS[r.workload].describe()}"


@pytest.mark.parametrize("name", sorted(WORKLOADS))
def test_spots_lie_in_the_destination_windows(name):
    """The places the H100 suite plants special values: inside each name's window, some on every name."""
    tables, geom, *_ = compiled(name)
    w = WORKLOADS[name]
    found = spots(tables, geom)
    assert sorted(found) == list(range(len(w.pulls)))
    for i, coords in found.items():
        off, loc = w.pulls[i].dst
        assert coords and all(o <= c < o + n for coord in coords for c, o, n in zip(coord, off, loc))

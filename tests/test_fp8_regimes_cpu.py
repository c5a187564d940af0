"""The scaled-fp8 branch catalogue (tests/fp8_regimes.py) without a GPU: every named workload compiled on host
memory through the planner path of a direct pull, its tables replayed with the oracle interpreters and
compared with requantize / dequantize, and every regime shown to hold on its workload's tables."""

import functools

import numpy as np
import pytest
import torch

from oracle import dequant_fp8_oracle, requant_fp8_oracle
from tests import test_dequant_fp8_cpu as dq_cpu
from tests import test_requant_fp8_cpu as rq_cpu
from tests.fp8_regimes import ES, REGIMES, WORKLOADS, geometry
from tests.helpers import region

# Every regime the catalogue names.  A regime added there without a workload that reaches it, or dropped
# from it, fails test_catalogue_is_complete until this list says so too.
EXPECTED = [
    "rq_block_unit_all_vec", "rq_block_unit_byte_piece", "rq_block_unit_straddling_chunk",
    "rq_block_unit_piece_off_16_columns", "rq_block_unit_batch",
    "rq_band_vec_short_rows", "rq_band_vec_long_rows", "rq_band_byte_piece", "rq_band_one_row_at_stage_bound",
    "rq_band_over_128_rows", "rq_band_several_sources", "rq_band_source_scale_step", "rq_band_batch",
    "rq_tensor_tile_rows_vec", "rq_tensor_tile_rows_byte", "rq_tensor_tile_full_width",
    "rq_channel_long_rows_block_source", "rq_channel_long_rows_channel_source", "rq_two_pass_source_scale_step",
    "rq_two_pass_over_256_groups", "rq_tile_batch",
    "dq_vec0_bfloat16", "dq_vec1_bfloat16", "dq_vec0_float16", "dq_vec1_float16", "dq_vec0_float32", "dq_vec1_float32",
    "dq_vec0_aligned_source", "dq_tile_full_width", "dq_tile_column_remainder", "dq_tile_256_rows_channel",
    "dq_vec_tile_ragged_cols",
]


def test_catalogue_is_complete():
    assert sorted(REGIMES) == sorted(EXPECTED)
    assert {r.workload for r in REGIMES.values()} == set(WORKLOADS)  # every regime has a workload and vice versa
    for name, r in REGIMES.items():
        assert name.split("_")[0] == {"requant": "rq", "dequant": "dq"}[WORKLOADS[r.workload].kind], name


def inputs(w):
    return rq_cpu.fp8_full(w.shape, w.seed), rq_cpu.global_scale(w.sg, w.shape, w.seed)


@functools.lru_cache(maxsize=None)
def replayed(name):
    """Compile workload `name` on host memory, replay its tables, check them against the oracle and return
    (tables, Geometry).  The tables' addresses are stale afterwards: predicates only compare them."""
    w = WORKLOADS[name]
    q, s = inputs(w)
    (off, loc) = w.dst
    if w.kind == "requant":
        dest, dest_scale, tables, (_, _, arr, _, _) = rq_cpu.compile_pull(q, s, w.sg, list(w.src), w.dst, w.out)
        geom = geometry(dest.data_ptr(), loc, 1, arr, len(arr))
        requant_fp8_oracle.replay(*tables)
        want_q, want_s = requant_fp8_oracle.requantize(region(q, off, loc).view(torch.uint8).numpy(),
                                                       rq_cpu.local_scale(s, w.sg, off, loc).numpy(), w.sg, off[-2], off[-1], w.out)
        assert np.array_equal(dest.view(torch.uint8).numpy(), want_q), w.describe()
        assert rq_cpu.same_scale(dest_scale.numpy(), want_s), w.describe()
    else:
        dest, tables, (_, _, arr, _) = dq_cpu.compile_pull(q, s, w.sg, list(w.src), w.dst, dequant_fp8_oracle.DST[w.out])
        geom = geometry(dest.data_ptr(), loc, ES[w.out], arr, len(arr))
        dequant_fp8_oracle.replay(tables)
        want = dequant_fp8_oracle.dequantize(region(q, off, loc).view(torch.uint8).numpy(),
                                             dq_cpu.local_scale(s, w.sg, off, loc).numpy(), w.sg, off[-2], off[-1], w.out)
        assert np.array_equal(dq_cpu.torch_bits(dest), want), w.describe()
    return tables, geom


@pytest.mark.parametrize("name", sorted(WORKLOADS))
def test_workload_replays_to_the_oracle(name):
    replayed(name)


@pytest.mark.parametrize("regime", sorted(REGIMES))
def test_regime_is_hit_by_its_workload(regime):
    r = REGIMES[regime]
    tables, geom = replayed(r.workload)
    assert r.holds(tables, geom), f"{regime} ({r.doc}) not reached by {WORKLOADS[r.workload].describe()}"

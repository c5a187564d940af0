"""The fp8 cast edge workloads (tests/fp8_cast_regimes.py) without a GPU: compiled at every tile size of
the regime matrix, their rect tables must reach the tile boundaries, fp8 mover regimes and kernel kind
tests/test_gpu_fp8_cast_regimes.py relies on, and replayed through the fp8 oracle they must write what
the oracle writes for the same windows, byte for byte."""

import pytest
import torch

from oracle import fp8_oracle
from tests import fp8_cast_regimes as fr
from tests.helpers import KIND_BF16_E4M3, KIND_GENERIC, edge_coverage, plan_kind, rect_fields, rects_for
from torchstore_b200 import _native

KIND = {"fp8": KIND_GENERIC, "bf16_e4m3": KIND_BF16_E4M3, "fp8_mixed": KIND_GENERIC}


@pytest.fixture(autouse=True)
def _default_knobs(monkeypatch):
    for k in ("TSB_TILE_BYTES", "TSB_LINK", "TSB_LINK_STAGE_BYTES"):
        monkeypatch.delenv(k, raising=False)


def compiled(name, tile_units, seed=1):
    host = fr.materialise(fr.workload(name, tile_units), "cpu", seed, tile_units)
    rects, n = rects_for(host)
    table, tiles, info = _native.plan_compile_host(0, rects, n, 0, tile_units)
    return host, table, tiles, info


@pytest.mark.parametrize("name", fr.WORKLOADS)
@pytest.mark.parametrize("tile_units", fr.TILE_UNITS)
def test_workload_reaches_its_regimes(tile_units, name):
    _, table, _, info = compiled(name, tile_units)
    fields = rect_fields(table)
    assert plan_kind(fields) == KIND[name]
    assert info.num_link_tiles == 0
    missing = sorted(k for k, hit in edge_coverage(fields, tile_units).items() if not hit)
    assert not missing, missing
    modes = set(fields["mode"].tolist()) & set(fr.FP8_MODES)
    assert modes == ({26} if name == "bf16_e4m3" else set(fr.FP8_MODES))
    for mode, regimes in fr.mode_regimes(fields, tile_units).items():
        if mode in fr.FP8_VECTOR_MODES:  # every vector mover: a short last wide segment, N-D narrow rows over tiles
            assert all(regimes.values()), (mode, regimes)
    if name == "fp8_mixed":
        assert set(fields["mode"].tolist()) - set(fr.FP8_MODES)  # byte moves and 16-bit casts beside the fp8 ones


def test_mixed_workload_has_link_tiles_under_link_2(monkeypatch):
    monkeypatch.setenv("TSB_LINK", "2")
    for tile_units in fr.TILE_UNITS:
        _, table, _, info = compiled("fp8_mixed", tile_units)
        fields = rect_fields(table)
        assert info.num_link_tiles > 0 and info.num_tiles > 0
        assert set(fields[fields["link"] == 1]["mode"].tolist()) == {4}  # the link warp moves 16-byte units only
        for name in ("fp8", "bf16_e4m3"):
            assert compiled(name, tile_units)[3].num_link_tiles == 0


@pytest.mark.parametrize("name", fr.WORKLOADS)
@pytest.mark.parametrize("tile_units", fr.TILE_UNITS)
def test_replayed_tables_match_the_oracle(tile_units, name):
    """The whole destination allocation (window, the rest of its base and the slack behind it)."""
    cases = fr.workload(name, tile_units)
    direct = fr.materialise(cases, "cpu", 7, tile_units)
    rects, n = rects_for(direct)
    fp8_oracle.copy_rects(rects, n, nan_mode=1)
    replay, table, tiles, info = compiled(name, tile_units, seed=7)
    fp8_oracle.replay_plan(table, tiles, tile_units, nan_mode=1)
    for i, ((_, _, want, _), (_, _, got, _)) in enumerate(zip(direct, replay)):
        assert torch.equal(got.view(torch.uint8), want.view(torch.uint8)), (i, cases[i].src_dtype, cases[i].dst_dtype)

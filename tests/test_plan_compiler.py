"""Host logic of the plan compiler (csrc/plan.cu) checked on the CPU: the compiled tables
(DevRect/DevTile) are replayed on host memory by the oracle's interpreter, unit by unit with the
kernel's arithmetic, and must reproduce the oracle's direct rectangle copy bit for bit."""

import random

import numpy as np
import pytest
import torch

from oracle import c_oracle
from tests.helpers import (KIND_B16, KIND_F32_BF16, KIND_GENERIC, MODE_B16, VECTOR_CAST_MODES, bytes_of, edge_coverage,
                           edge_workload, materialise, plan_kind, random_case, rect_fields, rects_for)
from torchstore_b200 import _native


def _run(cases, seed, tile_units, flags=0):
    a = materialise(cases, "cpu", seed)
    b = materialise(cases, "cpu", seed)
    rects_a, n_a = rects_for(a)
    rects_b, n_b = rects_for(b)
    assert n_a == n_b
    c_oracle.copy_rects(rects_a, n_a, nan_mode=0)
    table, tiles, info = _native.plan_compile_host(0, rects_b, n_b, flags, tile_units)
    assert info.num_tiles + info.num_link_tiles == tiles.shape[0]
    c_oracle.replay_plan(table, tiles, info.tile_bytes // 16, nan_mode=0)
    for (sa, da, dbase_a, _), (sb, db, dbase_b, _) in zip(a, b):
        assert np.array_equal(bytes_of(dbase_a), bytes_of(dbase_b))
    return a, info, table


@pytest.mark.parametrize("tile_units", [64, 256, 4096])
@pytest.mark.parametrize("cast", [False, True])
@pytest.mark.parametrize("link", ["1", "2"])
def test_compiled_plan_replays_to_oracle_result(tile_units, cast, link, monkeypatch):
    # TSB_LINK=2 routes every eligible 16-byte-unit rect through the link queue (small tiles, one
    # ring stage each); the interpreter also checks what a link tile may look like
    monkeypatch.setenv("TSB_LINK", link)
    rng = random.Random(100 + tile_units + cast)
    cases = [random_case(rng, cast=cast) for _ in range(60)]
    _run(cases, seed=5, tile_units=tile_units)


@pytest.mark.parametrize("tile_units", [64, 256, 4096, 32768])
@pytest.mark.parametrize("workload", ["mixed", "cast", "b16", "f32_bf16"])
@pytest.mark.parametrize("link", ["1", "2"])
def test_edge_workloads_replay_to_oracle_result(tile_units, workload, link, monkeypatch):
    """Edge-biased windows (tests/helpers.edge_workload) at every copy tile size the kernel is run
    with: the compiled tables reach the boundaries they aim at and replay to the oracle's bytes."""
    monkeypatch.setenv("TSB_LINK", link)
    rng = random.Random(f"edge-{tile_units}-{workload}")
    if workload in ("b16", "f32_bf16"):
        cases = edge_workload(rng, tile_units, uniform=workload)
    else:
        cases = edge_workload(rng, tile_units, cast=workload == "cast")
    _, info, table = _run(cases, seed=11, tile_units=tile_units)
    f = rect_fields(table)
    assert info.tile_bytes == tile_units * 16
    if workload == "b16":
        assert plan_kind(f) == KIND_B16
    elif workload == "f32_bf16":
        assert plan_kind(f) == KIND_F32_BF16
    else:
        assert plan_kind(f) == KIND_GENERIC
    if workload == "cast":
        assert set(f["mode"].tolist()) & set(VECTOR_CAST_MODES)
        assert set(f["mode"].tolist()) & {9, 11, 13, 15, 17, 19, 20, 21}  # scalar casts
    if workload == "mixed":
        assert MODE_B16 in f["mode"] and (f["mode"] < MODE_B16).any()
    if link == "1":
        cov = edge_coverage(f, tile_units)
        missing = sorted(k for k, hit in cov.items() if not hit)
        assert not missing, missing
    elif workload in ("mixed", "b16"):  # only 16-byte-unit moves ride the link warp
        assert info.num_link_tiles > 0 and f["link"].any()


def test_same_dtype_result_equals_torch_copy():
    """The oracle's rectangle copy is torch's dst.copy_(src) (what the reference executes)."""
    rng = random.Random(7)
    cases = [random_case(rng) for _ in range(40)]
    a, _, _ = _run(cases, seed=9, tile_units=256)
    ref = materialise(cases, "cpu", 9)
    for (s, d, dbase, _), (rs, rd, rbase, _) in zip(a, ref):
        rd.copy_(rs)
        assert np.array_equal(bytes_of(dbase), bytes_of(rbase))


def test_tile_order_interleaves_sources_and_covers_everything(monkeypatch):
    # 3 "sources" (devices 1,2,3) feeding device 0, equal sizes: tiles must rotate 1,2,3,1,2,3...
    # (copy queue: TSB_LINK=0 keeps NVLink sources with the copy warps)
    monkeypatch.setenv("TSB_LINK", "0")
    src = [torch.arange(64 * 1024, dtype=torch.int32) + i for i in range(3)]
    dst = torch.zeros(3, 64 * 1024, dtype=torch.int32)
    from torchstore_b200.planner import StridedMem, build_rects

    pairs = []
    for i in range(3):
        s = StridedMem.from_tensor(src[i])
        s = StridedMem(s.ptr, s.shape, s.stride, s.dtype, device=i + 1)
        pairs.append((s, StridedMem.from_tensor(dst[i])))
    rects, n = build_rects(pairs)
    table, tiles, info = _native.plan_compile_host(0, rects, n, 0, 256)
    assert info.num_rects == 3 and info.payload_bytes == 3 * 256 * 1024
    assert info.remote_src_bytes == info.src_bytes
    order = tiles[:, 0].tolist()
    assert order[:6] == [0, 1, 2, 0, 1, 2]
    # every (rect, tile) exactly once
    seen = set(map(tuple, tiles.tolist()))
    assert len(seen) == tiles.shape[0] == 3 * 64
    c_oracle.replay_plan(table, tiles, 256)
    for i in range(3):
        assert torch.equal(dst[i], src[i])
    # NO_INTERLEAVE keeps rect order
    _, tiles2, _ = _native.plan_compile_host(0, rects, n, _native.TSB_PLAN_NO_INTERLEAVE, 256)
    assert tiles2[:, 0].tolist() == sorted(tiles2[:, 0].tolist())
    # default: NVLink sources ride the link queue -- 4 KiB tiles, rotated in granules of 8 (one claim)
    monkeypatch.delenv("TSB_LINK")
    dst.zero_()
    table, tiles, info = _native.plan_compile_host(0, rects, n, 0, 256)
    assert info.num_tiles == 0 and info.num_link_tiles == 3 * 64 and info.link_bytes == info.remote_src_bytes
    assert info.block == 256 + 32
    assert tiles[:, 0].tolist()[:32] == [0] * 8 + [1] * 8 + [2] * 8 + [0] * 8
    assert len(set(map(tuple, tiles.tolist()))) == 3 * 64
    c_oracle.replay_plan(table, tiles, 256)
    for i in range(3):
        assert torch.equal(dst[i], src[i])


def test_vector_mode_selection_and_alignment_fallbacks():
    base = torch.zeros(4096 + 64, dtype=torch.uint8)
    out = torch.zeros(4096 + 64, dtype=torch.uint8)
    off = (-base.data_ptr()) % 16
    off_o = (-out.data_ptr()) % 16
    from torchstore_b200.planner import StridedMem, build_rects

    def mode_of(src_off, dst_off, n):
        s = StridedMem(base.data_ptr() + off + src_off, (n,), (1,), torch.uint8, -1)
        d = StridedMem(out.data_ptr() + off_o + dst_off, (n,), (1,), torch.uint8, -1)
        rects, k = build_rects([(s, d)])
        table, _, info = _native.plan_compile_host(0, rects, k, 0, 256)
        return int(table.view(np.uint32)[(16 + 96 + 24) // 4 + 6]), info  # DevRect.mode

    assert mode_of(0, 0, 1024)[0] == 4  # 16-byte units
    assert mode_of(8, 0, 1024)[0] == 3
    assert mode_of(4, 8, 1024)[0] == 2
    assert mode_of(2, 0, 1024)[0] == 1
    assert mode_of(1, 0, 1024)[0] == 0
    assert mode_of(0, 0, 1000)[0] == 3  # 1000 % 16 != 0 -> 8-byte units
    assert mode_of(0, 0, 1024)[1].num_vector_rects == 1


def test_empty_and_degenerate_rects():
    from torchstore_b200.planner import StridedMem, build_rects

    a = torch.arange(12, dtype=torch.float32).reshape(3, 4)
    b = torch.zeros(3, 4)
    # empty window is skipped by the planner
    rects, n = build_rects([(StridedMem.from_tensor(a[:0]), StridedMem.from_tensor(b[:0]))])
    assert n == 0
    table, tiles, info = _native.plan_compile_host(0, rects, n, 0, 64)
    assert info.num_tiles == 0
    # 0-d tensor
    s, d = torch.tensor(3.5), torch.tensor(0.0)
    rects, n = build_rects([(StridedMem.from_tensor(s), StridedMem.from_tensor(d))])
    table, tiles, info = _native.plan_compile_host(0, rects, n, 0, 64)
    c_oracle.replay_plan(table, tiles, 64)
    assert d.item() == 3.5
    # single column (innermost stride != itemsize): element-granular path
    rects, n = build_rects([(StridedMem.from_tensor(a[:, 1]), StridedMem.from_tensor(b[:, 2]))])
    table, tiles, info = _native.plan_compile_host(0, rects, n, 0, 64)
    c_oracle.replay_plan(table, tiles, 64)
    assert torch.equal(b[:, 2], a[:, 1]) and b[:, :2].abs().sum() == 0


def test_unsupported_cast_is_rejected():
    from torchstore_b200.planner import StridedMem, build_rects

    a = torch.zeros(8, dtype=torch.int32)
    b = torch.zeros(8, dtype=torch.float32)
    with pytest.raises(NotImplementedError):
        build_rects([(StridedMem.from_tensor(a), StridedMem.from_tensor(b))])


def test_unequal_sources_are_spread_proportionally(monkeypatch):
    """A small remote share in the COPY queue (link queue off) must be spread over the whole launch,
    not bunched at the front."""
    from torchstore_b200.planner import StridedMem, build_rects

    monkeypatch.setenv("TSB_LINK", "0")

    big = torch.zeros(5 * 64 * 1024, dtype=torch.int32)   # local: 5x the tiles
    small = torch.zeros(64 * 1024, dtype=torch.int32)     # remote
    out_b, out_s = torch.zeros_like(big), torch.zeros_like(small)
    sb = StridedMem.from_tensor(big)
    ss = StridedMem.from_tensor(small)
    pairs = [(StridedMem(sb.ptr, sb.shape, sb.stride, sb.dtype, device=0), StridedMem.from_tensor(out_b)),
             (StridedMem(ss.ptr, ss.shape, ss.stride, ss.dtype, device=1), StridedMem.from_tensor(out_s))]
    rects, n = build_rects(pairs)
    _, tiles, info = _native.plan_compile_host(0, rects, n, 0, 256)
    order = tiles[:, 0]
    assert (order == 1).sum() == 64 and (order == 0).sum() == 320
    pos = np.nonzero(order == 1)[0]
    gaps = np.diff(pos)
    assert gaps.min() >= 5 and gaps.max() <= 7  # one remote tile every ~6 tiles, start to finish
    assert pos[0] <= 6 and pos[-1] >= len(order) - 7


def test_oracle_threaded_copy_equals_single_threaded():
    """bench.py's cpu_baseline uses the oracle's pthread driver; it must move exactly the same bytes
    as the single-threaded path (row-balanced partition across rect boundaries)."""
    rng = random.Random(77)
    cases = [random_case(rng, cast=(i % 3 == 0), max_elems=1 << 18) for i in range(40)]
    # a few big contiguous ones so that total bytes >> 1 MiB and partitions cut inside rects
    a = materialise(cases, "cpu", 3)
    big_src = torch.arange(1 << 21, dtype=torch.int32)
    big_a = torch.zeros_like(big_src)
    a.append((big_src.reshape(2048, 1024)[:, 100:900], big_a.reshape(2048, 1024)[:, 100:900], big_a, big_src))
    ra, na = rects_for(a)
    c_oracle.copy_rects(ra, na, nan_mode=0, nthreads=1)
    for threads in (2, 7, 16):
        # re-materialise the destinations so untouched bytes match too
        b2 = materialise(cases, "cpu", 3)
        big_c = torch.zeros_like(big_src)
        b2.append((big_src.reshape(2048, 1024)[:, 100:900], big_c.reshape(2048, 1024)[:, 100:900], big_c, big_src))
        r2, n2 = rects_for(b2)
        c_oracle.copy_rects(r2, n2, nan_mode=0, nthreads=threads)
        for (_, _, da, _), (_, _, d2, _) in zip(a, b2):
            assert np.array_equal(bytes_of(da), bytes_of(d2)), threads

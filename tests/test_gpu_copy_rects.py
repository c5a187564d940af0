"""GPU parity of the copy_rects kernel through the C-ABI: identical rectangle descriptors are run by
the CUDA kernel (on device copies) and by the C oracle (on host copies) and compared byte for byte,
including the bytes OUTSIDE every destination window."""

import os
import random

import numpy as np
import pytest
import torch

from oracle import c_oracle
from tests.helpers import (CAST_PAIRS, assert_equal_modulo_nan, bytes_of, materialise, native_session, random_case,
                           rects_for)
from torchstore_b200 import _native
from torchstore_b200.planner import StridedMem, build_rects

pytestmark = pytest.mark.gpu
_init = pytest.fixture(scope="module", autouse=True)(native_session)


def run_product(pairs, device=0, flags=0):
    # the plan runs on the library's copy stream, which is not ordered after torch's stream: the
    # sources and destinations torch just wrote must be complete first
    torch.cuda.synchronize()
    rects, n = rects_for(pairs)
    plan = _native.plan_create(device, rects, n, flags)
    info = _native.plan_info(plan)
    before = _native.launch_count()
    _native.plan_run(plan, None)
    _native.stream_sync(device, None)
    assert _native.launch_count() == before + (1 if info.num_tiles or info.num_link_tiles else 0)
    _native.plan_destroy(plan)
    return info


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("cast", [False, True])
@pytest.mark.parametrize("force_generic", [False, True])
@pytest.mark.parametrize("link", ["default", "all"])
def test_random_rects_match_oracle(seed, cast, force_generic, link, monkeypatch):
    """link="all" (TSB_LINK=2) routes every 16-byte-unit rect through the link warp's TMA bulk ring
    even though the sources are local, so the NVLink data path is parity-tested on one GPU."""
    if force_generic:
        monkeypatch.setenv("TSB_FORCE_GENERIC", "1")
    else:
        monkeypatch.delenv("TSB_FORCE_GENERIC", raising=False)
    if link == "all":
        monkeypatch.setenv("TSB_LINK", "2")
    else:
        monkeypatch.delenv("TSB_LINK", raising=False)
    rng = random.Random(1000 * seed + cast)
    cases = [random_case(rng, cast=cast, max_elems=1 << 18) for _ in range(80)]
    host = materialise(cases, "cpu", seed)
    dev = materialise(cases, "cuda:0", seed)
    rects, n = rects_for(host)
    c_oracle.copy_rects(rects, n, nan_mode=1)
    run_product(dev)
    for (hs, hd, hbase, _), (ds, dd, dbase, _), case in zip(host, dev, cases):
        # window and everything around it
        assert_equal_modulo_nan(dbase, hbase, cast=case.src_dtype != case.dst_dtype)


@pytest.mark.parametrize("src_dtype,dst_dtype", CAST_PAIRS)
def test_cast_matches_torch_cuda_bit_exact(src_dtype, dst_dtype):
    """The cast path must equal what the reference computes on a GPU-resident param:
    tensor.to(transfer_dtype) on CUDA (direct_weight_sync.py:133), NaNs included."""
    gen = torch.Generator().manual_seed(3)
    n = 1 << 20
    raw = torch.randint(0, 256, (n * src_dtype.itemsize,), dtype=torch.uint8, generator=gen).view(src_dtype).cuda()
    # add edge values
    edge = torch.tensor([0.0, -0.0, 1.0, float("inf"), float("-inf"), float("nan"), 65504.0, 65520.0, 1e-8, 3.3895e38],
                        dtype=torch.float64).to(src_dtype).cuda()
    src = torch.cat([edge, raw])[: n - (n % 8)]
    want = src.to(dst_dtype)
    got = torch.zeros_like(want)
    run_product([(src, got)])
    if dst_dtype == torch.float32 and src_dtype == torch.float64:
        assert_equal_modulo_nan(got, want, cast=True)  # x86/CUDA differ in NaN payload propagation only
    else:
        assert torch.equal(got.view(torch.uint8), want.view(torch.uint8))
    # scalar path (misaligned views)
    got2 = torch.zeros(want.numel() + 1, dtype=dst_dtype, device="cuda")[1:]
    run_product([(src, got2)])
    assert_equal_modulo_nan(got2, want, cast=True)


def test_large_contiguous_int32_is_bit_exact():
    """Config #2 shape in miniature (1 GiB): integer/index tensors must be bit-exact."""
    n = 1 << 28
    src = torch.arange(n, dtype=torch.int32, device="cuda")
    dst = torch.zeros_like(src)
    info = run_product([(src, dst)])
    assert info.payload_bytes == n * 4 and info.num_vector_rects == 1
    assert torch.equal(src, dst)
    # properties at full size: sum of a checksum of checksums
    assert int(dst.view(torch.int64).sum().item()) == int(src.view(torch.int64).sum().item())


@pytest.fixture(params=["default", "all"])
def link_mode(request, monkeypatch):
    """"all" = TSB_LINK=2: the link warp (TMA bulk ring) moves every 16-byte-unit rect."""
    if request.param == "all":
        monkeypatch.setenv("TSB_LINK", "2")
    else:
        monkeypatch.delenv("TSB_LINK", raising=False)
    return request.param


def test_narrow_row_reshard_shapes(link_mode):
    """wo / w2 style rectangles: 512 x 512 and 512 x 1792 bf16 windows with 8 KiB / 28 KiB source
    pitch, written into a [4096, 512] / [4096, 1792] destination (SURVEY section 7.3)."""
    for cols_total, cols in ((4096, 512), (14336, 1792)):
        srcs = [torch.randn(512, cols_total, device="cuda").to(torch.bfloat16) for _ in range(8)]
        for r in (0, 3, 7):
            dst = torch.zeros(4096, cols, dtype=torch.bfloat16, device="cuda")
            pairs = [(srcs[s][:, r * cols:(r + 1) * cols], dst[s * 512:(s + 1) * 512]) for s in range(8)]
            info = run_product(pairs)
            assert info.num_vector_rects == 8
            assert (info.num_link_tiles > 0 and info.num_tiles == 0) if link_mode == "all" else info.num_link_tiles == 0
            want = torch.cat([s[:, r * cols:(r + 1) * cols] for s in srcs], dim=0)
            assert torch.equal(dst, want)


@pytest.mark.parametrize("stage_bytes,stages", [(8192, 6), (4096, 3), (16384, 4), (1024, 8)])
def test_link_ring_geometries(stage_bytes, stages, monkeypatch):
    """Every ring geometry the plan compiler accepts moves the same bytes: wide rows cut into stage-sized
    segments, narrow rows packed several per stage, strided destinations (per-row stores) and
    contiguous ones (one store per stage), 3-D wide rects, and a copy-queue rect beside them."""
    monkeypatch.setenv("TSB_LINK", "2")
    monkeypatch.setenv("TSB_LINK_STAGE_BYTES", str(stage_bytes))
    monkeypatch.setenv("TSB_LINK_STAGES", str(stages))
    g = torch.Generator(device="cuda").manual_seed(stage_bytes + stages)

    def rnd(*shape):
        return torch.randint(-30000, 30000, shape, dtype=torch.int16, device="cuda", generator=g)

    a = rnd(300, 1100)[:, :1004]  # rows of 2008 B, pitch 2200 B -> 8-byte units: stays in the copy queue
    b = rnd(1 << 21)         # one wide row (4 MiB)
    c = rnd(777, 4096)       # narrow 1 KiB windows, source pitch 8 KiB, destination contiguous
    d = rnd(64, 3, 20000)    # wide rows (16 KiB windows of 40 KB rows) under two outer dims
    e = rnd(512, 1792 * 8)   # 3.5 KiB windows into a strided destination
    e_dst = torch.zeros(512, 4096, dtype=torch.int16, device="cuda")
    outs = [torch.zeros(300, 1004, dtype=torch.int16, device="cuda"), torch.zeros_like(b), torch.zeros(777, 512, dtype=torch.int16, device="cuda"),
            torch.zeros(64, 3, 8192, dtype=torch.int16, device="cuda")]
    pairs = [(a, outs[0]), (b, outs[1]), (c[:, 1024:1536], outs[2]), (d[:, :, 4096:12288], outs[3]),
             (e[:, 1792:3584], e_dst[:, 1024:2816])]
    info = run_product(pairs)
    assert info.link_tile_bytes == stage_bytes and info.link_stages == stages
    assert info.num_link_tiles > 0 and info.num_tiles > 0
    assert torch.equal(outs[0], a) and torch.equal(outs[1], b)
    assert torch.equal(outs[2], c[:, 1024:1536]) and torch.equal(outs[3], d[:, :, 4096:12288])
    assert torch.equal(e_dst[:, 1024:2816], e[:, 1792:3584])
    assert int(e_dst[:, :1024].abs().sum()) == 0 and int(e_dst[:, 2816:].abs().sum()) == 0


def test_fenced_launch_poll_and_elapsed():
    """tsb_plan_launch: fence-in on the caller's stream, kernel, fence-out -- torch work queued before
    is seen by the copy and torch work queued after sees the copy, with no host wait in between."""
    a = torch.zeros(1 << 24, dtype=torch.int32, device="cuda")
    b = torch.zeros_like(a)
    rects, n = build_rects([(StridedMem.from_tensor(a), StridedMem.from_tensor(b))])
    plan = _native.plan_create(0, rects, n)
    assert _native.plan_poll(plan)  # never launched: trivially done
    for i in range(1, 4):
        a.fill_(i)  # queued on torch's stream, not waited for
        _native.plan_launch(plan, _native.torch_stream(0))
        c = b + 0   # torch stream waits for the done event
        _native.plan_wait(plan)
        assert _native.plan_poll(plan)
        assert _native.plan_elapsed_ms(plan) > 0
        assert int(c.min()) == i and int(c.max()) == i
    _native.plan_destroy(plan)


def test_one_shot_tables_come_from_a_recycled_pool():
    a = torch.arange(1 << 16, dtype=torch.int64, device="cuda")
    outs = [torch.zeros_like(a) for _ in range(40)]
    before = _native.pool_stats()
    for o in outs:
        rects, n = build_rects([(StridedMem.from_tensor(a), StridedMem.from_tensor(o))])
        _native.copy_rects(0, rects, n)
    _native.stream_sync(0, None)
    after = _native.pool_stats()
    assert all(torch.equal(a, o) for o in outs)
    # back-to-back calls may need a few blocks in flight at once, never one per call
    assert after["allocs"] - before["allocs"] <= 16
    assert after["reuses"] - before["reuses"] >= 24


def test_many_tiny_and_one_huge_in_one_launch(link_mode):
    tiny_src = [torch.randn(512, device="cuda").to(torch.bfloat16) for _ in range(300)]
    tiny_dst = [torch.zeros(512, dtype=torch.bfloat16, device="cuda") for _ in range(300)]
    big_src = torch.randn(64 << 20, device="cuda").to(torch.bfloat16)
    big_dst = torch.zeros_like(big_src)
    info = run_product(list(zip(tiny_src, tiny_dst)) + [(big_src, big_dst)])
    assert info.num_rects == 301
    assert torch.equal(big_src, big_dst)
    assert all(torch.equal(a, b) for a, b in zip(tiny_src, tiny_dst))


def test_one_shot_copy_rects_and_events():
    a = torch.arange(1 << 20, dtype=torch.int64, device="cuda")
    b = torch.zeros_like(a)
    rects, n = build_rects([(StridedMem.from_tensor(a), StridedMem.from_tensor(b))])
    torch.cuda.synchronize()
    start = _native.Event(0, timing=True).record(None)
    _native.copy_rects(0, rects, n)
    done = _native.Event(0, timing=True).record(None)
    done.synchronize()
    assert done.query()
    assert start.elapsed_ms(done) > 0
    assert torch.equal(a, b)


def test_caller_stream_and_torch_interop():
    """Launching on torch's current stream orders with torch work on that stream."""
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        a = torch.full((1 << 22,), 7, dtype=torch.int32, device="cuda")
        b = torch.zeros_like(a)
        rects, n = build_rects([(StridedMem.from_tensor(a), StridedMem.from_tensor(b))])
        plan = _native.plan_create(0, rects, n)
        _native.plan_run(plan, s.cuda_stream)
        c = b + 1
    s.synchronize()
    assert int(c.sum().item()) == 8 * (1 << 22)
    _native.plan_destroy(plan)


def test_arena_alloc_free_ring():
    arena = _native.arena_create(0, 64 << 20)
    st = _native.arena_stats(arena)
    assert st.capacity == 64 << 20 and st.in_use == 0
    ptrs = [_native.arena_alloc(arena, 1 << 20) for _ in range(32)]
    assert len(set(ptrs)) == 32 and all(p % 256 == 0 for p in ptrs)
    assert _native.arena_stats(arena).in_use == 32 << 20
    for p in ptrs[::2]:
        _native.arena_free(arena, p)
    big = _native.arena_alloc(arena, 30 << 20)  # fits only in the untouched tail
    with pytest.raises(_native.TsbError):
        _native.arena_alloc(arena, 40 << 20)
    _native.arena_free(arena, big)
    for p in ptrs[1::2]:
        _native.arena_free(arena, p)
    assert _native.arena_stats(arena).in_use == 0
    whole = _native.arena_alloc(arena, 64 << 20)  # everything coalesced back
    _native.arena_free(arena, whole)
    # arena memory is exportable and usable by the kernel
    p = _native.arena_alloc(arena, 1 << 20)
    reg = _native.export_region(p, 1 << 20)
    assert reg.nbytes == 1 << 20 and _native.import_region(reg, 0) == p
    _native.arena_destroy(arena)


def test_export_import_same_process_torch_suballocation():
    """A tensor carved by torch's caching allocator exports as (allocation handle, offset)."""
    pad = torch.empty(1000, device="cuda")  # noqa: F841 -- make the next tensor a sub-allocation
    t = torch.arange(4096, dtype=torch.float32, device="cuda")
    reg = _native.export_region(t.data_ptr(), t.numel() * 4)
    assert reg.nbytes == 4096 * 4 and reg.alloc_bytes >= reg.offset + reg.nbytes
    assert _native.import_region(reg, 0) == t.data_ptr()
    blob = _native.region_to_bytes(reg)
    assert len(blob) == 120 and _native.region_from_bytes(blob).offset == reg.offset


"""The fp8 casts on the H100: every bf16/f16/f32 pattern narrowed to float8_e4m3fn and float8_e5m2
bit for bit like torch's CUDA .to() (NaN encodings included), every fp8 pattern widened, random
multi-rect fp8 workloads against the C oracle, direct weight sync with fp8 staging and fp8
destinations, and the store path's fused fp8 gets."""

import json
import os
import random

import pytest
import torch

import torchstore_b200 as ts
import workloads
from oracle import fp8_oracle
from tests.helpers import (DEV, E4M3, GUARD, assert_equal_modulo_nan, assert_same_bits_or_nan, cleanup, named,
                           native_session, rect_fields, register_boxes, run, sha256_of, shard_box)
from tests.test_fp8_cast_cpu import SHORT as SHORT_NAMES
from tests.test_fp8_cast_cpu import VECTOR_MODE, fp8_case, host_bases
from torchstore_b200 import _native
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource
from torchstore_b200.planner import StridedMem, build_rects
from torchstore_b200.transport.types import TensorSlice

pytestmark = pytest.mark.gpu
E5M2 = torch.float8_e5m2
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "direct_fp8.json")
_init = pytest.fixture(scope="module", autouse=True)(native_session)


def u8(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous().view(torch.uint8)


def guarded_pitched(shape, dtype, lead: int, pitch_pad: int = 0):
    """A destination window of `shape` inside a guard-filled buffer: `lead` elements before the window's
    first element, rows `pitch_pad` elements longer than the window's."""
    rows, cols = shape
    pitch = cols + pitch_pad
    base = torch.full(((rows * pitch + lead + 64) * dtype.itemsize,), GUARD, dtype=torch.uint8, device=DEV).view(dtype)
    win = base[lead: lead + rows * pitch].view(rows, pitch)[:, :cols]
    return base, win


def layouts(src_flat: torch.Tensor, dst_dtype):
    """(name, src window, dst window, dst base) over the same elements: one contiguous vector run, the
    same one element off alignment (scalar), strided narrow rows and strided wide rows."""
    n = src_flat.numel()
    out = []
    base, win = guarded_pitched((1, n), dst_dtype, 16 // dst_dtype.itemsize * 2 if dst_dtype.itemsize < 16 else 2)
    out.append(("vector", src_flat.view(1, n), win, base))
    base, win = guarded_pitched((1, n), dst_dtype, 1)
    out.append(("scalar", src_flat.view(1, n), win, base))
    for name, cols in (("narrow", 64), ("wide", 65536)):
        if n % cols:
            continue
        rows = n // cols
        spad = 16
        sbase = torch.empty(rows * (cols + spad), dtype=src_flat.dtype, device=DEV)
        swin = sbase.view(rows, cols + spad)[:, :cols]
        swin.copy_(src_flat.view(rows, cols))
        base, win = guarded_pitched((rows, cols), dst_dtype, 16, pitch_pad=16)
        out.append((name, swin, win, base))
    return out


def run_pairs(pairs, expect_modes=None):
    torch.cuda.synchronize()
    rects, n = build_rects([(StridedMem.from_tensor(s), StridedMem.from_tensor(d)) for s, d in pairs])
    if expect_modes is not None:
        table, _, _ = _native.plan_compile_host(0, rects, n)
        assert set(rect_fields(table)["mode"].tolist()) == expect_modes
    plan = _native.plan_create(0, rects, n)
    try:
        _native.plan_run(plan, _native.torch_stream(0))
        torch.cuda.synchronize()
        return _native.plan_info(plan)
    finally:
        _native.plan_destroy(plan)


def check_guards(base: torch.Tensor, win: torch.Tensor):
    mask = torch.ones(base.numel(), dtype=torch.bool, device=DEV)
    offs = (win.data_ptr() - base.data_ptr()) // base.element_size()
    rows, cols = win.shape
    pos = offs + torch.arange(rows, device=DEV)[:, None] * win.stride(0) + torch.arange(cols, device=DEV)[None, :]
    mask[pos.reshape(-1)] = False
    outside = u8(base).view(-1, base.element_size())[mask]
    assert bool((outside == GUARD).all()), "a byte outside the destination window changed"


@pytest.mark.parametrize("src_dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("dst_dtype", [E4M3, E5M2])
@pytest.mark.parametrize("force_generic", [False, True])
def test_every_16_bit_pattern_narrows_like_torch(src_dtype, dst_dtype, force_generic, monkeypatch):
    if force_generic:
        monkeypatch.setenv("TSB_FORCE_GENERIC", "1")
    else:
        monkeypatch.delenv("TSB_FORCE_GENERIC", raising=False)
    pats = torch.arange(-32768, 32768, dtype=torch.int32, device=DEV).to(torch.int16).view(src_dtype)
    src = torch.cat([pats, pats])  # 2 x 65536: one wide row each in the "wide" layout
    want = src.to(dst_dtype)
    vmode = VECTOR_MODE[(src_dtype, dst_dtype)]
    for name, swin, dwin, dbase in layouts(src, dst_dtype):
        run_pairs([(swin, dwin)], expect_modes={vmode + 1} if name == "scalar" else {vmode})
        assert torch.equal(u8(dwin), u8(want.view(dwin.shape))), (name, force_generic)
        check_guards(dbase, dwin)


@pytest.mark.parametrize("dst_dtype", [E4M3, E5M2])
def test_every_f32_pattern_narrows_like_torch(dst_dtype):
    """All 2^32 f32 patterns in chunks of 2^28, generated and compared on the device, on a vector and a
    scalar layout."""
    chunk = 1 << 28
    idx = torch.arange(chunk, dtype=torch.int32, device=DEV)
    bits = torch.empty_like(idx)
    src = bits.view(torch.float32)
    vmode = VECTOR_MODE[(torch.float32, dst_dtype)]
    plans = []
    for name, lead in (("vector", 16), ("scalar", 1)):
        base, win = guarded_pitched((1, chunk), dst_dtype, lead)
        rects, n = build_rects([(StridedMem.from_tensor(src.view(1, chunk)), StridedMem.from_tensor(win))])
        table, _, _ = _native.plan_compile_host(0, rects, n)
        assert set(rect_fields(table)["mode"].tolist()) == ({vmode} if name == "vector" else {vmode + 1})
        plans.append((_native.plan_create(0, rects, n), win, base, lead))
    stream = _native.torch_stream(0)
    try:
        for k in range(16):
            torch.add(idx, -(1 << 31) + k * chunk, out=bits)
            want = u8(src.to(dst_dtype))
            for plan, win, base, lead in plans:
                _native.plan_run(plan, stream)  # ordered after the rewrite and before the compare by torch's stream
                assert torch.equal(u8(win).view(-1), want), k
                b = u8(base)
                assert bool((b[:lead] == GUARD).all()) and bool((b[lead + chunk:] == GUARD).all())
            del want
        torch.cuda.synchronize()
    finally:
        for plan, *_ in plans:
            _native.plan_destroy(plan)


@pytest.mark.parametrize("src_dtype", [E4M3, E5M2])
@pytest.mark.parametrize("dst_dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_every_fp8_pattern_widens_like_torch(src_dtype, dst_dtype):
    pats = torch.arange(256, dtype=torch.int32, device=DEV).to(torch.uint8).view(src_dtype)
    src = pats.repeat(512)  # 131072 elements: narrow rows of 64 and two wide rows
    want = src.to(dst_dtype)
    vmode = VECTOR_MODE[(src_dtype, dst_dtype)]
    for name, swin, dwin, dbase in layouts(src, dst_dtype):
        run_pairs([(swin, dwin)], expect_modes={vmode + 1} if name == "scalar" else {vmode})
        with named(name):
            assert_same_bits_or_nan(dwin.reshape(-1), want)
        check_guards(dbase, dwin)


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("force_generic", [False, True])
def test_random_fp8_workloads_match_the_oracle(seed, force_generic, monkeypatch):
    if force_generic:
        monkeypatch.setenv("TSB_FORCE_GENERIC", "1")
    else:
        monkeypatch.delenv("TSB_FORCE_GENERIC", raising=False)
    rng = random.Random(9000 + seed)
    cases = [fp8_case(rng, edge=i % 2 == 1) for i in range(60)]
    host = host_bases(cases, seed)
    rects, n = build_rects([(StridedMem.from_tensor(p[0]), StridedMem.from_tensor(p[1])) for p in host])
    fp8_oracle.copy_rects(rects, n, nan_mode=1)
    dev = [tuple(t.to(DEV) if i >= 2 else None for i, t in enumerate(p)) for p in host_bases(cases, seed)]
    pairs = [(c.src_view(d[3]), c.dst_view(d[2])) for c, d in zip(cases, dev)]
    run_pairs(pairs)
    bad = []
    for c, (sv, dv, want, _), d, (dsrc, ddst) in zip(cases, host, dev, pairs):
        try:
            assert_equal_modulo_nan(d[2], want, cast=True)
        except AssertionError:
            r, k = build_rects([(StridedMem.from_tensor(dsrc), StridedMem.from_tensor(ddst))])
            f = rect_fields(_native.plan_compile_host(0, r, k)[0])
            g, w = u8(d[2].cpu()).view(-1), u8(want).view(-1)
            first = int((g != w).nonzero()[0]) if bool((g != w).any()) else -1
            bad.append((SHORT_NAMES[c.src_dtype], SHORT_NAMES[c.dst_dtype], tuple(sv.shape), sv.stride(), dv.stride(),
                        sv.storage_offset(), dv.storage_offset(), f[["mode", "n_outer", "rows", "units_per_row", "wide"]].tolist(),
                        first, hex(int(g[first])) if first >= 0 else None, hex(int(w[first])) if first >= 0 else None))
    assert not bad, bad


# ---- direct weight sync -------------------------------------------------------------------------------
def direct_fp8_full(gshape, src_dtype, seed):
    """Same values as oracle/gen_golden_fp8.py direct_fp8_full (the fixture's global tensors)."""
    g = torch.Generator().manual_seed(seed)
    full = torch.randn(gshape, generator=g) * 2.0 ** torch.randint(-12, 12, gshape, generator=g).float()
    full.view(-1)[::97] *= 7e4
    return full.to(getattr(torch, src_dtype))


def tslice(shape, n, r, placement):
    off, loc = workloads.shard_box(shape, n, r, placement)
    return TensorSlice(off, (r,), tuple(shape), loc, (n,))


def box(t, ts_):
    return t[tuple(slice(o, o + s) for o, s in zip(ts_.offsets, ts_.local_shape))]


def test_register_fp8_transfer_dtype_and_pull_matches_torch_and_the_reference():
    with open(GOLDEN) as f:
        cases = json.load(f)["cases"]
    assert len(cases) >= 6
    for c in cases:
        full = direct_fp8_full(tuple(c["global_shape"]), c["src_dtype"], c["seed"])
        fdt = getattr(torch, c["transfer_dtype"])
        sources, handles = register_boxes(full, [shard_box(full.shape, c["n_src"], r, 0) for r in range(c["n_src"])],
                                          transfer_dtype=fdt)
        want_full = full.to(DEV).to(fdt)
        for drank, rec in c["dest"].items():
            dsl = tslice(full.shape, c["n_dst"], int(drank), tuple(c["dst_placement"]))
            dest = torch.zeros(dsl.local_shape, dtype=fdt, device=DEV)
            sync = DirectWeightSyncDest()
            run(sync.pull({"w": handles}, {"w": dest}, {"w": dsl}))
            assert torch.equal(u8(dest), u8(box(want_full, dsl))), (c, drank)
            assert sha256_of(dest) == rec["sha256"], (c, drank)
            sync.close()
        cleanup(sources)


@pytest.mark.parametrize("src_dtype", [torch.bfloat16, torch.float32])
def test_refresh_after_an_in_place_update(src_dtype):
    full = direct_fp8_full((128, 96), str(src_dtype).replace("torch.", ""), 7)
    sources, handles = register_boxes(full, [shard_box(full.shape, 4, r, 0) for r in range(4)], transfer_dtype=E4M3)
    dsl = tslice(full.shape, 2, 1, ("S", 1))
    dest = torch.zeros(dsl.local_shape, dtype=E4M3, device=DEV)
    sync = DirectWeightSyncDest()
    run(sync.pull({"w": handles}, {"w": dest}, {"w": dsl}))
    for src, shard, _ in sources:
        shard.mul_(-3.0)
        assert src.refresh() == 1
    run(sync.pull({"w": handles}, {"w": dest}, {"w": dsl}))
    want = box((full.to(DEV) * -3.0).to(src_dtype).to(E4M3), dsl)
    assert torch.equal(u8(dest), u8(want))
    sync.close()


@pytest.mark.parametrize("dst_dtype", [E4M3, E5M2])
def test_bf16_handles_into_fp8_destinations_fuse_the_cast_into_the_gather(dst_dtype):
    full = direct_fp8_full((256, 128), "bfloat16", 11)
    _, handles = register_boxes(full, [shard_box(full.shape, 4, r, 0) for r in range(4)])
    for drank in range(2):
        dsl = tslice(full.shape, 2, drank, ("S", 1))
        dest = torch.zeros(dsl.local_shape, dtype=dst_dtype, device=DEV)
        sync = DirectWeightSyncDest()
        before = _native.launch_count()
        run(sync.pull({"w": handles}, {"w": dest}, {"w": dsl}))
        assert _native.launch_count() == before + 1
        assert torch.equal(u8(dest), u8(box(full.to(DEV).to(dst_dtype), dsl)))
        sync.close()


@pytest.mark.parametrize("src_fp8", [E4M3, E5M2])
def test_fp8_handles_into_bf16_destinations(src_fp8):
    full = direct_fp8_full((256, 128), "bfloat16", 12).to(src_fp8)
    _, handles = register_boxes(full, [shard_box(full.shape, 4, r, 0) for r in range(4)])
    dsl = tslice(full.shape, 2, 0, ("S", 1))
    dest = torch.zeros(dsl.local_shape, dtype=torch.bfloat16, device=DEV)
    sync = DirectWeightSyncDest()
    run(sync.pull({"w": handles}, {"w": dest}, {"w": dsl}))
    assert_same_bits_or_nan(dest.reshape(-1), box(full.to(DEV).to(torch.bfloat16), dsl).reshape(-1))
    sync.close()


def test_transfer_dtype_without_a_fused_cast_is_refreshed_like_the_reference():
    """An int64 buffer and a float64 param with transfer_dtype=float8_e4m3fn: the reference stages
    them with local.to(transfer_dtype) and refreshes with staging.copy_(source); so does this."""
    sd = {"w": torch.randn(64, 64, device=DEV).to(torch.bfloat16),
          "steps": torch.arange(-40, 40, dtype=torch.int64, device=DEV) * 9,
          "scale": torch.randn(32, dtype=torch.float64, device=DEV) * 300}
    src = DirectWeightSyncSource()
    handles = src.register(sd, rank=0, transfer_dtype=E4M3)
    assert all(h.rdma_buffer.dtype == E4M3 for h in handles.values())
    assert len(src._refresh_plans) == 1 and len(src._copied) == 2
    dest = {k: torch.zeros(v.shape, dtype=E4M3, device=DEV) for k, v in sd.items()}
    sync = DirectWeightSyncDest()
    run(sync.pull({k: [h] for k, h in handles.items()}, dest))
    for k in sd:
        assert torch.equal(u8(dest[k]), u8(sd[k].to(E4M3))), k
    sd["steps"].add_(5)
    sd["scale"].mul_(-1)
    sd["w"].mul_(2)
    assert src.refresh() == 3
    run(sync.pull({k: [h] for k, h in handles.items()}, dest))
    for k in sd:
        assert torch.equal(u8(dest[k]), u8(sd[k].to(E4M3))), k
    sync.close()
    run(src.cleanup())


def test_put_and_get_state_dict_direct_rdma_with_fp8_transfer_dtype():
    import torch.distributed as dist
    from torch.testing._internal.distributed.fake_pg import FakeStore

    async def main():
        dist.init_process_group("fake", store=FakeStore(), rank=0, world_size=1)
        await ts.initialize()
        try:
            src = {"w": torch.randn(256, 128, device=DEV).to(torch.bfloat16), "b": torch.randn(128, device=DEV) * 1e3}
            await ts.put_state_dict(src, "policy_fp8", direct_rdma=True, transfer_dtype=E4M3)
            dst = {k: torch.zeros(v.shape, dtype=E4M3, device=DEV) for k, v in src.items()}
            out = await ts.get_state_dict("policy_fp8", user_state_dict=dst, direct_rdma=True)
            assert out is dst
            for k in src:
                assert torch.equal(u8(dst[k]), u8(src[k].to(E4M3))), k
            src["w"].mul_(0.5)
            await ts.put_state_dict(None, "policy_fp8", direct_rdma=True, transfer_dtype=E4M3)
            await ts.get_state_dict("policy_fp8", user_state_dict=dst, direct_rdma=True)
            assert torch.equal(u8(dst["w"]), u8(src["w"].to(E4M3)))
        finally:
            await ts.shutdown()
            dist.destroy_process_group()

    run(main())


# ---- store path ---------------------------------------------------------------------------------------
@pytest.fixture
def _store_env(monkeypatch):
    monkeypatch.delenv("RANK", raising=False)
    monkeypatch.setenv("LOCAL_RANK", "0")
    monkeypatch.delenv("TORCHSTORE_B200_GET_DEVICE", raising=False)
    yield


@pytest.mark.parametrize("dst_dtype", [E4M3, E5M2])
def test_store_get_batch_into_fp8_destinations_is_fused_and_replayed(dst_dtype, _store_env):
    async def main():
        await ts.initialize()
        try:
            lane = (await ts.client()).fast_lane
            src = {f"k{i}": direct_fp8_full((96 + i, 80), "bfloat16", 20 + i).to(DEV) for i in range(4)}
            await ts.put_batch(src)
            dst = {k: torch.zeros(v.shape, dtype=dst_dtype, device=DEV) for k, v in src.items()}
            before = _native.launch_count()
            await ts.get_batch(dst)  # slow path: one fused launch, recorded
            assert _native.launch_count() == before + 1
            for k in src:  # the same bytes as torch's copy_
                assert torch.equal(u8(dst[k]), u8(torch.empty_like(dst[k]).copy_(src[k]))), k
            for k in src:
                src[k].mul_(-0.25)
            await ts.put_batch(src)
            hits = lane.get_hits
            before = _native.launch_count()
            out = await ts.get_batch(dst)  # replayed by the fast lane
            assert lane.get_hits == hits + 1 and _native.launch_count() == before + 1
            assert all(out[k] is dst[k] for k in dst)
            for k in src:
                assert torch.equal(u8(dst[k]), u8(torch.empty_like(dst[k]).copy_(src[k]))), k
        finally:
            await ts.shutdown()

    run(main())

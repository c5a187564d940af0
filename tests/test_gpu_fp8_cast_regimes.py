"""copy_rects' plain fp8 casts in the regimes tests/test_gpu_fp8.py never reaches: the fp8 edge workloads
(tests/fp8_cast_regimes.py) under every tile size, capped grid, static scheduling, forced generic kernel
and link setting of the regime matrix; the KIND_BF16_E4M3 kernel and a mixed fp8 plan around the
boundary between a CTA's static and claimed tiles and across pipelined relaunches; fp8 windows past
2^32 bytes; and a bf16 FSDP -> fp8 TP weight sync at model scale.

Every test compares the whole destination allocation (the bytes around each window included) with the
fp8 oracle or torch's CUDA .to() -- fp8 outputs byte for byte, widened outputs with any NaN equal to
any NaN -- and asserts from plan_info and the compiled rect table that it reached the regime it is
named for."""

import numpy as np
import pytest
import torch

from oracle import fp8_oracle
from oracle import reshard_oracle as ro
from tests import fp8_cast_regimes as fr
from tests.helpers import (DEV, E4M3, KERNEL_REGIMES, KIND_BF16_E4M3, KIND_GENERIC, MODE_B16, assert_equal_modulo_nan,
                           assert_same_bits_or_nan, compiled, edge_coverage, llama_layout, native_session, plan_kind,
                           rect_fields, rects_for, run, run_plan, set_knobs)
from tests.test_fp8_cast_cpu import VECTOR_MODE
from torchstore_b200 import _native
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource
from torchstore_b200.planner import StridedMem, build_rects
from torchstore_b200.transport.types import TensorSlice

pytestmark = pytest.mark.gpu
E5M2 = torch.float8_e5m2
BF16, F16, F32 = torch.bfloat16, torch.float16, torch.float32
GUARD = fr.GUARD
_init = pytest.fixture(scope="module", autouse=True)(native_session)


def assert_same(got: torch.Tensor, want: torch.Tensor):
    """On the device: fp8 (and byte) tensors byte for byte, wider floats with any NaN equal to any NaN."""
    if got.element_size() == 1:
        assert got.dtype == want.dtype and torch.equal(got.view(torch.uint8), want.view(torch.uint8)), \
            int((got.view(torch.uint8) != want.view(torch.uint8)).sum())
    else:
        assert_same_bits_or_nan(got, want)


def guarded_flat(n: int, dtype) -> torch.Tensor:
    """A flat destination allocation of n elements, every byte GUARD."""
    return torch.full((n * dtype.itemsize,), GUARD, dtype=torch.uint8, device=DEV).view(dtype)


def expected(windows, allocs):
    """Clones of the destination allocations with torch's CUDA .to() of each source in its window.
    windows: [(src view, alloc -> dst view)] against allocs."""
    want = [a.clone() for a in allocs]
    for (src, win), w in zip(windows, want):
        win(w).copy_(src)
    return want


# ---- regime matrix ------------------------------------------------------------------------------------
def _check_regime(workload, tile_bytes, cap, sched, link, fields, hinfo, info):
    T = tile_bytes // 16
    assert (info.num_tiles, info.num_link_tiles) == (hinfo.num_tiles, hinfo.num_link_tiles)
    assert info.tile_bytes == tile_bytes
    assert plan_kind(fields) == (KIND_BF16_E4M3 if workload == "bf16_e4m3" else KIND_GENERIC)
    work = max(info.num_tiles, -(-info.num_link_tiles // 8))
    if cap is None:
        assert info.grid >= min(work, torch.cuda.get_device_properties(0).multi_processor_count)
    else:
        assert info.grid == cap and work > 3 * cap  # TSB_MAX_GRID reached the launch; CTAs go past their static tiles
    if sched == "static":
        assert info.num_link_tiles == 0
        if cap is not None:
            assert info.num_tiles > 3 * info.grid  # the stride fallback runs
    if workload == "fp8_mixed" and link == 2:
        assert info.num_link_tiles > 0 and info.num_tiles > 0
        assert set(fields[fields["link"] == 1]["mode"].tolist()) == {MODE_B16}
        return
    assert info.num_link_tiles == 0
    missing = sorted(k for k, hit in edge_coverage(fields, T).items() if not hit)
    assert not missing, missing
    for mode, regimes in fr.mode_regimes(fields, T).items():
        if mode in fr.FP8_VECTOR_MODES:
            assert all(regimes.values()), (mode, regimes)


@pytest.mark.parametrize("workload", fr.WORKLOADS)
@pytest.mark.parametrize("tile_bytes", [1024, 4096, 65536, 524288])
def test_fp8_edge_workloads_match_oracle_across_regimes(tile_bytes, workload, monkeypatch):
    """The fp8 edge workload of this tile size materialised once and run by the fp8 oracle once, then run
    by the product into fresh copies of the destination allocations under each regime of this tile size,
    both as a compiled plan (tsb_plan_run) and one-shot (tsb_copy_rects)."""
    T = tile_bytes // 16
    cases = fr.workload(workload, T)
    seed = tile_bytes % 1009
    host = fr.materialise(cases, "cpu", seed, T)
    hrects, hn = rects_for(host)
    fp8_oracle.copy_rects(hrects, hn, nan_mode=1)
    dev = fr.materialise(cases, DEV, seed, T)
    initial = [d[2].clone() for d in dev]
    regimes = [r for r in KERNEL_REGIMES if r[0] == tile_bytes]
    assert {r[1] for r in regimes} == {None, 1, 5}
    for _, cap, sched, generic, link in regimes:
        set_knobs(monkeypatch, TSB_TILE_BYTES=tile_bytes, TSB_MAX_GRID=cap, TSB_LINK=link,
                  TSB_STATIC_SCHED=1 if sched == "static" else None, TSB_FORCE_GENERIC=1 if generic else None)
        for one_shot in (False, True):
            outs = [a.clone() for a in initial]
            pairs = [(d[0], fr.dst_window(c, o)) for d, c, o in zip(dev, cases, outs)]
            rects, n, fields, hinfo = compiled(pairs)
            if one_shot:
                _native.copy_rects(0, rects, n, stream=_native.torch_stream(0))
                torch.cuda.synchronize()
            else:
                info = run_plan(rects, n)
                _check_regime(workload, tile_bytes, cap, sched, link, fields, hinfo, info)
            for i, (out, (_, _, want, _), c) in enumerate(zip(outs, host, cases)):
                try:
                    assert_equal_modulo_nan(out, want, cast=c.src_dtype != c.dst_dtype)
                except AssertionError:
                    raise AssertionError((cap, sched, generic, link, one_shot, i, c.src_dtype, c.dst_dtype))


# ---- static / claimed tile boundary -------------------------------------------------------------------
SLACK = 4096  # bytes behind every allocation: more than one 1 KiB tile of the widest unit


def _stack(dtype, rows, m, width, g):
    """A flat allocation holding a [rows, m + 1, width] stack and the slack behind it; random bits."""
    n = rows * (m + 1) * width
    raw = torch.randint(0, 256, ((n * dtype.itemsize + SLACK),), dtype=torch.uint8, device=DEV, generator=g)
    return raw.view(dtype), lambda a: a[:n].view(rows, m + 1, width)


def _boundary_plan(plan, ntiles, g):
    """(windows, dst allocs) of a plan of 1 KiB tiles (64 units) with `ntiles` copy tiles: a wide
    row of 3 tiles and a 5-unit segment, then narrow rows (8 per tile) under two outer dims whose last
    tile is ragged.  The N-D rect sits in a stack whose outer dim holds every row, so a mover that
    addresses its rows by the outer stride alone stays inside the allocation."""
    m = 4 * (ntiles - 4) - 1  # 2m rows: ntiles - 4 tiles of 8 rows, the last one of 6
    L = (3 * 64 + 5) * 16
    if plan == "bf16_e4m3":
        (wide_s, wide_d), (nd_s, nd_d), nd_w, (s0, d0) = (BF16, E4M3), (BF16, E4M3), 128, (8, 16)
    else:  # a vector f32 -> e5m2 row, then scalar e4m3 -> bf16 rows one element off alignment
        (wide_s, wide_d), (nd_s, nd_d), nd_w, (s0, d0) = (F32, E5M2), (E4M3, BF16), 8, (1, 3)
    a = torch.randint(0, 256, (L * wide_s.itemsize + 64 + SLACK,), dtype=torch.uint8, device=DEV, generator=g)
    a = a.view(wide_s)
    out_a = guarded_flat(L + 64 + SLACK, wide_d)
    b, bstack = _stack(nd_s, 2 * m, m, nd_w + 16, g)
    out_b = guarded_flat((2 * m * (m + 1) * (nd_w + 32) * nd_d.itemsize + SLACK) // nd_d.itemsize, nd_d)
    bdst = lambda o: o[: 2 * m * (m + 1) * (nd_w + 32)].view(2 * m, m + 1, nd_w + 32)
    # the wide row 16 bytes in on both sides; the N-D window: 2 of the stack's outer rows, m of m + 1
    sa = 16 // wide_s.itemsize
    windows = [(a[sa:sa + L], lambda o: o[16 // wide_d.itemsize:16 // wide_d.itemsize + L]),
               (bstack(b)[:2, :m, s0:s0 + nd_w], lambda o: bdst(o)[:2, :m, d0:d0 + nd_w])]
    return windows, [out_a, out_b]


@pytest.mark.parametrize("plan", ["bf16_e4m3", "generic"])
@pytest.mark.parametrize("sched", ["dynamic", "static"])
@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_fp8_tile_counts_around_the_static_claimed_boundary(plan, sched, delta, monkeypatch):
    """A grid of 3 with 3*grid-1, 3*grid and 3*grid+1 fp8 copy tiles: the last static tile, the first
    claimed (or strided) one, a wide row's short last segment and a rect-to-rect (and, in the generic
    plan, vector-to-scalar mode) header change between them."""
    cap = 3
    set_knobs(monkeypatch, TSB_TILE_BYTES=1024, TSB_MAX_GRID=cap, TSB_LINK=1,
              TSB_STATIC_SCHED=1 if sched == "static" else None)
    ntiles = 3 * cap + delta
    g = torch.Generator(device=DEV).manual_seed(60 + delta)
    windows, allocs = _boundary_plan(plan, ntiles, g)
    want = expected(windows, allocs)
    rects, n, fields, _ = compiled([(s, w(o)) for (s, w), o in zip(windows, allocs)])
    modes = fields["mode"].tolist()
    if plan == "bf16_e4m3":
        assert modes == [26, 26] and plan_kind(fields) == KIND_BF16_E4M3
    else:
        assert modes == [VECTOR_MODE[(F32, E5M2)], VECTOR_MODE[(E4M3, BF16)] + 1] and plan_kind(fields) == KIND_GENERIC
    assert fields["wide"].tolist() == [1, 0] and fields["n_outer"].tolist()[1] == 2
    assert int(fields["units_per_row"][0]) % 64 == 5 and int(fields["rows"][1]) % int(fields["split"][1]) != 0
    info = run_plan(rects, n)
    assert info.num_tiles == ntiles and info.grid == cap and info.num_link_tiles == 0
    for got, w in zip(allocs, want):
        assert_same(got, w)


# ---- pipelined relaunch -------------------------------------------------------------------------------
def _slacked(shape, dtype, guard: bool):
    """(flat allocation, alloc -> [shape] view of its front) with SLACK bytes behind; GUARD-filled or empty."""
    n = int(np.prod(shape))
    count = n + SLACK // dtype.itemsize
    a = guarded_flat(count, dtype) if guard else torch.empty(count, dtype=dtype, device=DEV)
    return a, lambda o: o[:n].view(shape)


def _relaunch_plan(kind, g):
    """(live sources, windows, dst allocs, rewrite) of a plan with more copy tiles than 3 per CTA of a
    full grid at 1 KiB tiles.  bf16_e4m3: wide bf16 rows with a short last segment and narrow N-D rows.
    mixed: vector f32 -> e4m3 rows, vector e5m2 -> f32 rows, scalar f16 -> e5m2 rows and 16-byte int32
    rows (link tiles under TSB_LINK=2).  rewrite(live, i) writes launch i's sources with torch ops."""
    if kind == "bf16_e4m3":
        m = 63
        bases = [torch.randn(1024, 1104, device=DEV, generator=g).to(BF16),
                 torch.randn(2 * m, m + 1, 144, device=DEV, generator=g).to(BF16)]
        src_dtypes = [BF16, BF16]
        dsts = [((1024, 1120), E4M3), ((2 * m, m + 1, 160), E4M3)]
        sw = [(slice(None), slice(8, 8 + 1088)), (slice(0, 2), slice(0, m), slice(8, 136))]
        dw = [(slice(None), slice(16, 16 + 1088)), (slice(0, 2), slice(0, m), slice(16, 144))]

        def rewrite(live, i):
            for b, lv in zip(bases, live):
                torch.mul(b, float(i + 1), out=lv)
    else:
        bases = [torch.randn(600, 1632, device=DEV, generator=g), torch.randn(300, 1056, device=DEV, generator=g) * 64,
                 torch.randn(256, 200, device=DEV, generator=g).to(F16),
                 torch.randint(-2**31, 2**31 - 1, (2048, 1024), dtype=torch.int32, device=DEV, generator=g)]
        src_dtypes = [F32, E5M2, F16, torch.int32]
        dsts = [((600, 1648), E4M3), ((300, 1040), F32), ((256, 144), E5M2), ((2048, 520), torch.int32)]
        sw = [(slice(None), slice(8, 1608)), (slice(None), slice(16, 1040)), (slice(None), slice(1, 129)),
              (slice(None), slice(256, 768))]
        dw = [(slice(None), slice(16, 1616)), (slice(None), slice(4, 1028)), (slice(None), slice(3, 131)),
              (slice(None), slice(4, 516))]

        def rewrite(live, i):
            torch.mul(bases[0], float(i + 1), out=live[0])
            live[1].copy_(bases[1] * float(i + 1))  # the e5m2 of a new f32 value per launch
            torch.mul(bases[2], float(i + 1), out=live[2])
            torch.bitwise_xor(bases[3], i * 104729, out=live[3])
    # sources too have slack behind them: a wide row may end at their last element
    live = [view(a) for a, view in (_slacked(b.shape, dt, False) for b, dt in zip(bases, src_dtypes))]
    allocs, views = zip(*(_slacked(shape, dt, True) for shape, dt in dsts))
    windows = [(lambda lv, ws=ws: lv[ws], lambda o, v=v, wd=wd: v(o)[wd]) for ws, wd, v in zip(sw, dw, views)]
    return live, windows, list(allocs), rewrite


@pytest.mark.parametrize("cap", [None, 3])
def test_pipelined_fp8_relaunches_see_new_sources_and_rearm_the_scheduler(cap, monkeypatch):
    """Ten tsb_plan_launch calls each of a KIND_BF16_E4M3 plan and a mixed fp8 plan, interleaved on
    torch's stream with no host wait: before each launch torch rewrites the sources, after it the
    destinations are cloned on the same stream.  Every snapshot must equal torch's .to() of its own
    launch's sources -- which a launch whose scheduler was not re-armed by the previous one misses."""
    set_knobs(monkeypatch, TSB_LINK=2, TSB_TILE_BYTES=1024, TSB_MAX_GRID=cap)
    g = torch.Generator(device=DEV).manual_seed(23)
    plans = []
    for kind in ("bf16_e4m3", "mixed"):
        live, windows, allocs, rewrite = _relaunch_plan(kind, g)
        init = [a.clone() for a in allocs]
        rects, n, fields, _ = compiled([(s(lv), w(a)) for lv, (s, w), a in zip(live, windows, allocs)])
        plan = _native.plan_create(0, rects, n)
        info = _native.plan_info(plan)
        assert info.num_tiles > 3 * info.grid
        assert info.grid == cap if cap else info.grid > 3
        if kind == "bf16_e4m3":
            assert plan_kind(fields) == KIND_BF16_E4M3 and info.num_link_tiles == 0
            assert fields["wide"].tolist() == [1, 0] and int(fields["n_outer"][1]) == 2
            assert int(fields["units_per_row"][0]) % 64 != 0
        else:
            assert plan_kind(fields) == KIND_GENERIC and info.num_link_tiles > 0
            assert fields["mode"].tolist() == [VECTOR_MODE[(F32, E4M3)], VECTOR_MODE[(E5M2, F32)],
                                               VECTOR_MODE[(F16, E5M2)] + 1, MODE_B16]
        plans.append((plan, live, windows, allocs, init, rewrite, []))
    launches = 10
    torch.cuda.synchronize()
    stream = _native.torch_stream(0)
    for i in range(launches):
        for k, (plan, live, _, allocs, _, rewrite, snaps) in enumerate(plans):
            rewrite(live, k * launches + i)
            _native.plan_launch(plan, stream)
            snaps.append([a.clone() for a in allocs])
    torch.cuda.synchronize()
    for k, (plan, live, windows, _, init, rewrite, snaps) in enumerate(plans):
        for i, snap in enumerate(snaps):
            rewrite(live, k * launches + i)
            want = expected([(s(lv), w) for lv, (s, w) in zip(live, windows)], init)
            for got, w in zip(snap, want):
                assert_same(got, w)
        _native.plan_destroy(plan)


# ---- windows past 4 GiB -------------------------------------------------------------------------------
def test_fp8_windows_beyond_4_gib(monkeypatch):
    """Narrow rows whose window starts past 2^32 bytes of an 8.7 GB allocation and spans more than 2^32
    bytes of row stride: f32 -> e4m3 and bf16 -> e5m2 from such a source, e4m3 -> f32 and e5m2 -> bf16
    with the fp8 source there, each in its vector and scalar layout."""
    set_knobs(monkeypatch)
    P, R, r0 = (1 << 20) + 16, 8300, 4100
    rows = R - r0
    g = torch.Generator(device=DEV).manual_seed(4)
    base = torch.randint(0, 256, (R * P,), dtype=torch.uint8, device=DEV, generator=g)
    cols = 4096
    srcs = {  # (window past 4 GiB, elements per row)
        (F32, E4M3): base.view(F32).view(R, P // 4)[r0:, 4:4 + cols // 4],
        (BF16, E5M2): base.view(BF16).view(R, P // 2)[r0:, 8:8 + cols // 2],
        (E4M3, F32): base.view(E4M3).view(R, P)[r0:, 16:16 + cols],
        (E5M2, BF16): base.view(E5M2).view(R, P)[r0:, 16:16 + cols],
    }
    for (sdt, ddt), win in srcs.items():
        want = win.to(ddt)
        w = win.shape[1]
        for vector in (True, False):
            start = 16 // ddt.itemsize if vector else 1
            out = guarded_flat(rows * (w + 2 * start + 16), ddt).view(rows, w + 2 * start + 16)
            rects, n, fields, _ = compiled([(win, out[:, start:start + w])])
            assert len(fields) == 1
            assert int(fields["mode"][0]) == VECTOR_MODE[(sdt, ddt)] + (0 if vector else 1)
            assert int(fields["src"][0]) - base.data_ptr() > 1 << 32
            assert int(fields["src_stride"][0][0]) * int(fields["rows"][0]) > 1 << 32
            if vector:
                assert int(fields["src_unit_bytes"][0]) == 16 * sdt.itemsize
            full = guarded_flat(out.numel(), ddt).view(out.shape)
            full[:, start:start + w] = want
            run_plan(rects, n)
            assert_same(out, full)
            del out, full
        del want
    del base, srcs
    torch.cuda.empty_cache()


# ---- at model scale -----------------------------------------------------------------------------------
def _box(t, sl):
    return t[tuple(slice(o, o + s) for o, s in zip(sl.offsets, sl.local_shape))]


@pytest.mark.parametrize("n", [1, 2, 4, 8])
def test_llama_bf16_fsdp_refresh_into_e4m3_and_tp_pulls_match_torch(n):
    """A scaled Llama-3 (2 layers, dims / 8) in bf16 FSDP(n) shards registered with
    transfer_dtype=float8_e4m3fn (the refresh plan is KIND_BF16_E4M3), pulled into e4m3 TP(n)
    destinations -- byte for byte torch's full.to(e4m3) sliced -- and then into bf16 TP(n) destinations,
    widening the same fp8 handles: torch's full.to(e4m3).to(bf16) sliced.  All ranks on one GPU."""
    layout = llama_layout(n_layers=2, scale=8)
    gen = torch.Generator().manual_seed(n)
    fulls = {k: (torch.randn(shape, generator=gen) * 2.0 ** torch.randint(-12, 9, shape, generator=gen).float()).to(BF16)
             for k, (shape, _) in layout.items()}
    want = {k: f.to(DEV).to(E4M3) for k, f in fulls.items()}
    sources, handles = [], {k: [] for k in layout}
    for r in range(n):
        sd, slices = {}, {}
        for name, (shape, _) in layout.items():
            sl = ro.make_slice(shape, (n,), (r,), [("S", 0)])
            sd[name] = _box(fulls[name], sl).contiguous().to(DEV)
            slices[name] = TensorSlice(sl.offsets, sl.coordinates, sl.global_shape, sl.local_shape, sl.mesh_shape)
        src = DirectWeightSyncSource()
        for name, h in src.register(sd, rank=r, transfer_dtype=E4M3, tensor_slices=slices).items():
            assert h.rdma_buffer.dtype == E4M3
            handles[name].append(h)
        assert not src._copied and len(src._staging) == len(layout)
        rects, k = build_rects([(StridedMem.from_tensor(local), StridedMem.from_tensor(staging))
                                for staging, local in src._staging.values()])
        assert plan_kind(rect_fields(_native.plan_compile_host(0, rects, k)[0])) == KIND_BF16_E4M3
        sources.append(src)
    for dtype in (E4M3, BF16):
        for drank in range(n):
            dest, dslices, boxes = {}, {}, {}
            for name, (shape, tp) in layout.items():
                dsl = ro.full_slice(shape) if n == 1 else ro.make_slice(shape, (n,), (drank,), [tp])
                dest[name] = torch.zeros(dsl.local_shape, dtype=dtype, device=DEV)
                if n > 1:
                    dslices[name] = TensorSlice(dsl.offsets, dsl.coordinates, dsl.global_shape, dsl.local_shape, dsl.mesh_shape)
                boxes[name] = dsl
            sync = DirectWeightSyncDest()
            run(sync.pull(handles, dest, dslices or None))
            for name in layout:
                assert_same(dest[name], _box(want[name], boxes[name]).to(dtype))
            sync.close()
    for src in sources:
        run(src.cleanup())

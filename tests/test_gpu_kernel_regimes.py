"""copy_rects parity in the regimes the random parity suite never reaches: non-default tile sizes,
static scheduling, capped grids (one CTA walking the whole queue; tile counts around the boundary
between a CTA's three static tiles and claimed ones), pipelined relaunches that need the scheduler
counters re-armed, every 16-bit and 32-bit cast source pattern, and offsets and splits past 32 bits.

Every test compares the whole destination allocation (the bytes around each window included) with
an independent reference, and asserts from plan_info and the compiled rect table that it reached the
regime it is named for."""

import random

import numpy as np
import pytest
import torch

from oracle import c_oracle
from tests.helpers import (KERNEL_REGIMES, KIND_B16, KIND_F32_BF16, KIND_GENERIC, MODE_B16, MODE_F32_BF16_V8,
                           VECTOR_CAST_MODES, assert_equal_modulo_nan, assert_same_bits_or_nan, compiled, edge_coverage,
                           edge_workload, materialise, native_session, plan_kind, rects_for, run_plan, set_knobs)
from torchstore_b200 import _native

pytestmark = pytest.mark.gpu

GUARD = 0xA5
_init = pytest.fixture(scope="module", autouse=True)(native_session)


# ---- regime matrix ------------------------------------------------------------------------------------
def _check_regime(workload, tile_bytes, cap, sched, link, fields, hinfo, info):
    T = tile_bytes // 16
    assert (info.num_tiles, info.num_link_tiles) == (hinfo.num_tiles, hinfo.num_link_tiles)
    assert info.tile_bytes == tile_bytes
    assert plan_kind(fields) == {"b16": KIND_B16, "f32_bf16": KIND_F32_BF16}.get(workload, KIND_GENERIC)
    work = max(info.num_tiles, -(-info.num_link_tiles // 8))
    if cap is None:
        assert info.grid >= min(work, torch.cuda.get_device_properties(0).multi_processor_count)
    else:
        assert info.grid == cap  # TSB_MAX_GRID reached the launch
        assert work > 3 * cap  # so CTAs go past their static tiles
    if sched == "static":
        assert info.num_link_tiles == 0  # static striding applies only without a link queue
        if cap is not None:
            assert info.num_tiles > 3 * info.grid  # the stride fallback runs
    if link == 1:
        assert info.num_link_tiles == 0
        missing = sorted(k for k, hit in edge_coverage(fields, T).items() if not hit)
        assert not missing, missing
    elif workload in ("mixed", "b16"):
        assert info.num_link_tiles > 0 and info.num_tiles > 0


@pytest.mark.parametrize("workload", ["mixed", "cast", "b16", "f32_bf16"])
@pytest.mark.parametrize("tile_bytes", [1024, 4096, 65536, 524288])
def test_edge_workloads_match_oracle_across_regimes(tile_bytes, workload, monkeypatch):
    """Edge-biased windows (tests/helpers.edge_workload) materialised once and run by the oracle once,
    then run by the product into fresh destination copies under each regime of this tile size, both as
    a compiled plan (tsb_plan_run) and one-shot (tsb_copy_rects)."""
    T = tile_bytes // 16
    rng = random.Random(f"regimes-{tile_bytes}-{workload}")
    if workload in ("b16", "f32_bf16"):
        cases = edge_workload(rng, T, uniform=workload)
    else:
        cases = edge_workload(rng, T, cast=workload == "cast")
    seed = tile_bytes % 1009
    host = materialise(cases, "cpu", seed)
    hrects, hn = rects_for(host)
    c_oracle.copy_rects(hrects, hn, nan_mode=1)
    dev = materialise(cases, "cuda:0", seed)
    initial = [d[2].clone() for d in dev]
    regimes = [r for r in KERNEL_REGIMES if r[0] == tile_bytes]
    assert {r[1] for r in regimes} == {None, 1, 5}
    for _, cap, sched, generic, link in regimes:
        set_knobs(monkeypatch, TSB_TILE_BYTES=tile_bytes, TSB_MAX_GRID=cap, TSB_LINK=link,
                  TSB_STATIC_SCHED=1 if sched == "static" else None, TSB_FORCE_GENERIC=1 if generic else None)
        for one_shot in (False, True):
            outs = [b.clone() for b in initial]
            pairs = [(d[0], c.dst_view(o)) for d, c, o in zip(dev, cases, outs)]
            rects, n, fields, hinfo = compiled(pairs)
            if one_shot:
                _native.copy_rects(0, rects, n, stream=_native.torch_stream(0))
                torch.cuda.synchronize()
            else:
                info = run_plan(rects, n)
                _check_regime(workload, tile_bytes, cap, sched, link, fields, hinfo, info)
            for out, (_, _, want, _), c in zip(outs, host, cases):
                assert_equal_modulo_nan(out, want, cast=c.src_dtype != c.dst_dtype)


@pytest.mark.parametrize("sched", ["dynamic", "static"])
@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_tile_counts_around_the_static_claimed_boundary(sched, delta, monkeypatch):
    """A grid of 3 with 3*grid-1, 3*grid and 3*grid+1 copy tiles: the last static tile, the first
    claimed (or strided) one, and rect-to-rect and mode-to-mode header changes between them."""
    cap = 3
    set_knobs(monkeypatch, TSB_TILE_BYTES=1024, TSB_MAX_GRID=cap, TSB_LINK=1,
              TSB_STATIC_SCHED=1 if sched == "static" else None)
    ntiles = 3 * cap + delta
    g = torch.Generator(device="cuda").manual_seed(40 + delta)
    a = torch.randint(0, 256, (4 * 1024 + 64,), dtype=torch.uint8, device="cuda", generator=g)
    b = torch.randint(0, 256, ((ntiles - 4) * 64 + 64,), dtype=torch.uint8, device="cuda", generator=g)
    out_a = torch.full_like(a, GUARD)
    out_b = torch.full_like(b, GUARD)
    # 4 tiles of 16-byte units, then odd-offset bytes (64 one-byte units per tile)
    pairs = [(a[16:16 + 4096], out_a[32:32 + 4096]), (b[1:1 + (ntiles - 4) * 64], out_b[3:3 + (ntiles - 4) * 64])]
    rects, n, fields, _ = compiled(pairs)
    assert fields["mode"].tolist() == [MODE_B16, 0]
    info = run_plan(rects, n)
    assert info.num_tiles == ntiles and info.grid == cap and info.num_link_tiles == 0
    want_a, want_b = torch.full_like(a, GUARD), torch.full_like(b, GUARD)
    want_a[32:32 + 4096] = a[16:16 + 4096]
    want_b[3:3 + (ntiles - 4) * 64] = b[1:1 + (ntiles - 4) * 64]
    assert torch.equal(out_a, want_a) and torch.equal(out_b, want_b)


# ---- pipelined relaunch -------------------------------------------------------------------------------
def _relaunch_workload(g):
    """Sources and destinations of a plan with copy tiles (8-byte-unit rows, a vector cast) and link
    tiles (16-byte-unit rows under TSB_LINK=2)."""
    srcs = [torch.randint(-2**31, 2**31 - 1, (1024, 1030), dtype=torch.int32, device="cuda", generator=g),
            torch.randint(-2**31, 2**31 - 1, (2048, 1024), dtype=torch.int32, device="cuda", generator=g),
            torch.randn(300, 2000, device="cuda", generator=g)]
    dsts = [torch.full((1024, 1040), -7, dtype=torch.int32, device="cuda"),
            torch.full((2048, 520), -7, dtype=torch.int32, device="cuda"),
            torch.full((300, 1616), -7.0, dtype=torch.bfloat16, device="cuda")]
    windows = [((slice(None), slice(2, 1026)), (slice(None), slice(8, 1032))),
               ((slice(None), slice(256, 768)), (slice(None), slice(4, 516))),
               ((slice(None), slice(8, 1608)), (slice(None), slice(8, 1608)))]
    return srcs, dsts, windows


def _rewrite(bases, live, i):
    """Launch-specific source data, written by torch ops on torch's stream."""
    torch.add(bases[0], i * 7919, out=live[0])
    torch.bitwise_xor(bases[1], i * 104729, out=live[1])
    torch.mul(bases[2], float(i + 1), out=live[2])


@pytest.mark.parametrize("cap", [None, 3])
def test_pipelined_relaunches_see_new_sources_and_rearm_the_scheduler(cap, monkeypatch):
    """Ten tsb_plan_launch calls of one plan on torch's stream with no host wait in between, a second
    plan interleaved: before each launch torch rewrites the sources, after it the destination is cloned
    on the same stream.  Every snapshot must hold its own launch's data -- including the link queue,
    which a launch that was not re-armed by the previous one would skip."""
    set_knobs(monkeypatch, TSB_LINK=2, TSB_TILE_BYTES=1024, TSB_MAX_GRID=cap)
    g = torch.Generator(device="cuda").manual_seed(17)
    bases_a, dsts_a, win_a = _relaunch_workload(g)
    bases_b, dsts_b, win_b = _relaunch_workload(g)
    live_a = [b.clone() for b in bases_a]
    live_b = [b.clone() for b in bases_b]
    init_a = [d.clone() for d in dsts_a]
    init_b = [d.clone() for d in dsts_b]

    def make(live, dsts, wins):
        pairs = [(s[ws], d[wd]) for s, d, (ws, wd) in zip(live, dsts, wins)]
        rects, n, fields, _ = compiled(pairs)
        plan = _native.plan_create(0, rects, n)
        return plan, _native.plan_info(plan), fields

    plan_a, info_a, fields_a = make(live_a, dsts_a, win_a)
    plan_b, info_b, _ = make(live_b, dsts_b, win_b)
    for info in (info_a, info_b):
        assert info.num_link_tiles > 0 and info.num_tiles > 3 * info.grid
        assert info.grid == cap if cap else info.grid > 3
    assert set(fields_a["mode"].tolist()) == {3, MODE_B16, MODE_F32_BF16_V8}
    launches = 10
    snaps_a, snaps_b = [], []
    torch.cuda.synchronize()
    stream = _native.torch_stream(0)
    for i in range(launches):
        _rewrite(bases_a, live_a, i)
        _native.plan_launch(plan_a, stream)
        snaps_a.append([d.clone() for d in dsts_a])
        _rewrite(bases_b, live_b, launches + i)
        _native.plan_launch(plan_b, stream)
        snaps_b.append([d.clone() for d in dsts_b])
    torch.cuda.synchronize()
    for bases, init, wins, snaps, off in ((bases_a, init_a, win_a, snaps_a, 0), (bases_b, init_b, win_b, snaps_b, launches)):
        live = [b.clone() for b in bases]
        for i, snap in enumerate(snaps):
            _rewrite(bases, live, off + i)
            for s, d0, (ws, wd), got in zip(live, init, wins, snap):
                want = d0.clone()
                want[wd].copy_(s[ws])
                assert torch.equal(got.view(torch.uint8), want.view(torch.uint8)), (off, i)
    _native.plan_destroy(plan_a)
    _native.plan_destroy(plan_b)


# ---- cast domains -------------------------------------------------------------------------------------
HALF_PAIRS = [(torch.bfloat16, torch.float32), (torch.float16, torch.float32),
              (torch.bfloat16, torch.float16), (torch.float16, torch.bfloat16)]


def _layouts(src, dst_dtype, device, strided=True):
    """(name, pairs, dst bases) for one flat source: the vector layout (16-byte aligned windows), the
    scalar layout (a destination one element off alignment) and strided 2-D windows with narrow and
    wide rows."""
    n = src.numel()
    vec = torch.full((n + 16,), GUARD, dtype=torch.uint8, device=device).to(dst_dtype)
    sca = vec.clone()
    out = [("vector", [(src, vec[8:8 + n])], [vec]), ("scalar", [(src, sca[1:1 + n])], [sca])]
    if not strided:
        return out
    # narrow rows (1000 elements) and wide rows (40000 elements: past one 64 KiB tile even as 8-element units)
    pairs, bases = [], []
    for rows, cols in ((64, 1000), (3, 40000)):
        flat = src if n >= rows * cols else src.repeat(-(-rows * cols // n))
        sb = torch.empty(rows, cols + 16, dtype=src.dtype, device=device)
        sb[:, 8:8 + cols].copy_(flat[: rows * cols].view(rows, cols))
        db = torch.full((rows, cols + 24), GUARD, dtype=torch.uint8, device=device).to(dst_dtype)
        pairs.append((sb[:, 8:8 + cols], db[:, 16:16 + cols]))
        bases.append(db)
    out.append(("strided", pairs, bases))
    return out


def _check_layout(name, fields, cast_pair):
    vmodes = set(fields["mode"].tolist()) & set(VECTOR_CAST_MODES)
    has_vector = torch.float64 not in cast_pair
    if name == "scalar" or not has_vector:
        assert not vmodes
    else:
        assert vmodes and len(set(fields["mode"].tolist())) == 1
    if name == "strided":
        assert sorted(fields["wide"].tolist()) == [0, 1] and (fields["n_outer"] == 1).all()


def _expected(pairs, bases):
    want = [b.clone() for b in bases]
    for (s, d), b, w in zip(pairs, bases, want):
        off = (d.data_ptr() - b.data_ptr()) // d.element_size()
        w.view(-1)[off:].as_strided(d.shape, d.stride()).copy_(s.to(d.dtype))
    return want


@pytest.mark.parametrize("src_dtype,dst_dtype", HALF_PAIRS)
def test_every_16_bit_source_pattern_casts_like_torch_and_the_oracle(src_dtype, dst_dtype):
    pats = torch.arange(1 << 16, dtype=torch.int32).view(torch.int16)[::2].contiguous().view(src_dtype)
    for (name, pairs, bases), (_, hpairs, hbases) in zip(_layouts(pats.cuda(), dst_dtype, "cuda"),
                                                         _layouts(pats, dst_dtype, "cpu")):
        rects, n, fields, _ = compiled(pairs)
        _check_layout(name, fields, (src_dtype, dst_dtype))
        want = _expected(pairs, bases)  # torch's CUDA .to()
        run_plan(rects, n)
        hrects, hn = rects_for(hpairs)
        c_oracle.copy_rects(hrects, hn, nan_mode=1)
        for got, w, o in zip(bases, want, hbases):
            assert_equal_modulo_nan(got, w, cast=True)
            assert_equal_modulo_nan(got, o, cast=True)


@pytest.mark.parametrize("dst_dtype", [torch.bfloat16, torch.float16, torch.float64])
def test_every_f32_pattern_casts_like_torch(dst_dtype):
    """All 2^32 f32 bit patterns in chunks of 2^28, generated on the device, compared on the device
    with torch's CUDA .to(): vector and scalar layouts, then strided narrow and wide rows once."""
    chunk = 1 << 28
    idx = torch.arange(chunk, dtype=torch.int32, device="cuda")
    bits = torch.empty_like(idx)
    src = bits.view(torch.float32)
    plans = []
    for name, pairs, bases in _layouts(src, dst_dtype, "cuda", strided=False):
        rects, n, fields, _ = compiled(pairs)
        _check_layout(name, fields, (torch.float32, dst_dtype))
        plans.append((_native.plan_create(0, rects, n), pairs, bases))
    guard = torch.full((16,), GUARD, dtype=torch.uint8, device="cuda").to(dst_dtype)
    stream = _native.torch_stream(0)
    for k in range(1 << 4):
        torch.add(idx, -(1 << 31) + k * chunk, out=bits)
        want = src.to(dst_dtype)
        for plan, [(_, d)], [base] in plans:
            _native.plan_run(plan, stream)  # ordered after the rewrite and before the compare by torch's stream
            assert_same_bits_or_nan(d, want)
            off = (d.data_ptr() - base.data_ptr()) // d.element_size()
            assert_same_bits_or_nan(base[:off], guard[:off])
            assert_same_bits_or_nan(base[off + chunk:], guard[: base.numel() - off - chunk])
        del want
    torch.cuda.synchronize()
    for plan, _, _ in plans:
        _native.plan_destroy(plan)
    del plans, idx, bits, src
    # strided narrow and wide rows over a random quarter-million patterns
    g = torch.Generator(device="cuda").manual_seed(5)
    rnd = torch.randint(-2**31, 2**31 - 1, (1 << 22,), dtype=torch.int32, device="cuda", generator=g).view(torch.float32)
    name, pairs, bases = _layouts(rnd, dst_dtype, "cuda")[2]
    rects, n, fields, _ = compiled(pairs)
    _check_layout(name, fields, (torch.float32, dst_dtype))
    want = _expected(pairs, bases)
    run_plan(rects, n)
    for got, w in zip(bases, want):
        assert_same_bits_or_nan(got, w)
    torch.cuda.empty_cache()


def _f64_to_f32_edges() -> np.ndarray:
    """f64 values where rounding to f32 goes wrong: exact f32 values, the midpoints between adjacent
    f32 values and one f64 ulp either side of them at every f32 exponent (subnormals included), the
    ties at FLT_MAX -> inf and at half the smallest subnormal -> 0, f64 subnormals, zeros,
    infinities and NaN payloads, all with both signs."""
    rng = np.random.default_rng(0)
    mants = np.concatenate([np.array([0, 1, 2, 3, 0x3FFFFF, 0x400000, 0x7FFFFE, 0x7FFFFF], np.uint32),
                            rng.integers(0, 1 << 23, 8, dtype=np.uint32)])
    a_bits = ((np.arange(255, dtype=np.uint32)[:, None] << 23) | mants[None, :]).reshape(-1)
    a_bits = a_bits[a_bits != 0x7F7FFFFF]  # FLT_MAX has no finite neighbour above: its tie is below
    a = a_bits.view(np.float32).astype(np.float64)
    b = (a_bits + 1).view(np.float32).astype(np.float64)
    mid = (a + b) / 2  # exact: 25 significant bits
    flt_max_tie = np.float64(2.0 ** 128 - 2.0 ** 103)
    half_min_sub = np.float64(2.0 ** -150)
    specials = np.array([flt_max_tie, half_min_sub, 3 * half_min_sub, np.float64(np.finfo(np.float32).max),
                         1e300, 1e-300, 0.0, np.inf], np.float64)
    vals = np.concatenate([a, mid, specials])
    vals = np.concatenate([vals, np.nextafter(vals, np.inf), np.nextafter(vals, -np.inf)])
    f64_bits = np.array([1, 2, 3, 0x0008000000000000, 0x000FFFFFFFFFFFFF, 0x7FF0000000000001, 0x7FF4000000000000,
                         0x7FF8000000000000, 0x7FF8000000000001, 0x7FFFFFFFFFFFFFFF], np.uint64)
    vals = np.concatenate([vals, f64_bits.view(np.float64)])
    vals = np.concatenate([vals, -vals])
    return vals[: len(vals) // 8 * 8]


def test_f64_to_f32_rounds_every_tie_like_numpy():
    x = _f64_to_f32_edges()
    assert len(x) > 40000
    src = torch.from_numpy(x).cuda()
    for name, pairs, bases in _layouts(src, torch.float32, "cuda"):
        rects, n, fields, _ = compiled(pairs)
        _check_layout(name, fields, (torch.float64, torch.float32))
        assert (fields["mode"] == 20).all()
        want = [b.cpu() for b in bases]
        for (s, d), b, w in zip(pairs, bases, want):
            with np.errstate(all="ignore"):  # overflow to inf and NaN quieting are part of the set
                ref = torch.from_numpy(s.cpu().numpy().astype(np.float32))
            off = (d.data_ptr() - b.data_ptr()) // 4
            w.view(-1)[off:].as_strided(d.shape, d.stride()).copy_(ref)
        run_plan(rects, n)
        for got, w in zip(bases, want):
            assert_equal_modulo_nan(got, w, cast=True)


# ---- offsets and splits past 32 bits ------------------------------------------------------------------
def test_odd_offset_byte_run_longer_than_2_30_splits_into_column_chunks():
    L = (1 << 30) + 12345
    g = torch.Generator(device="cuda").manual_seed(1)
    src = torch.randint(0, 256, (L + 64,), dtype=torch.uint8, device="cuda", generator=g)
    dst = torch.full((L + 16,), GUARD, dtype=torch.uint8, device="cuda")
    pairs = [(src[1:1 + L], dst[3:3 + L])]
    rects, n, fields, _ = compiled(pairs)
    assert fields["units_per_row"].tolist() == [1 << 30, L - (1 << 30)] and (fields["mode"] == 0).all()
    run_plan(rects, n)
    assert torch.equal(dst[3:3 + L], src[1:1 + L])
    assert bool((dst[:3] == GUARD).all()) and bool((dst[3 + L:] == GUARD).all())
    del src, dst
    torch.cuda.empty_cache()


def test_byte_column_of_more_than_2_30_rows_splits_into_row_halves():
    R = (1 << 30) + 1000
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.randint(0, 256, (2 * R,), dtype=torch.uint8, device="cuda", generator=g)
    y = torch.full((2 * R,), GUARD, dtype=torch.uint8, device="cuda")
    pairs = [(x.view(-1, 2)[:, 1], y.view(-1, 2)[:, 0])]
    rects, n, fields, _ = compiled(pairs)
    assert fields["rows"].tolist() == [R // 2, R - R // 2] and (fields["units_per_row"] == 1).all()
    assert (fields["magic"] == 0).all() and (fields["wide"] == 0).all()
    run_plan(rects, n)
    assert torch.equal(y.view(-1, 2)[:, 0], x.view(-1, 2)[:, 1])
    assert bool((y.view(-1, 2)[:, 1] == GUARD).all())  # the guard bytes interleave with the column
    del x, y
    torch.cuda.empty_cache()


@pytest.mark.parametrize("link", [1, 2])
def test_windows_beyond_4_gib(link, monkeypatch):
    """Narrow rows whose source window starts past 2^32 bytes and spans more than 2^32 bytes of row
    stride: a 16-byte-unit copy (through the link warp under TSB_LINK=2), and an f32->bf16 cast in its
    vector and scalar layouts."""
    set_knobs(monkeypatch, TSB_LINK=link)
    P, R, r0 = (1 << 20) + 16, 8300, 4100
    rows = R - r0
    g = torch.Generator(device="cuda").manual_seed(3)
    base = torch.randint(0, 256, (R * P,), dtype=torch.uint8, device="cuda", generator=g)
    win = base.view(R, P)[r0:, 16:16 + 4096]
    dst = torch.full((rows, 4096 + 32), GUARD, dtype=torch.uint8, device="cuda")
    rects, n, fields, _ = compiled([(win, dst[:, 16:16 + 4096])])
    assert len(fields) == 1 and fields["mode"][0] == MODE_B16
    assert int(fields["src"][0]) - base.data_ptr() > 1 << 32
    assert int(fields["src_stride"][0][0]) * int(fields["rows"][0]) > 1 << 32
    assert int(fields["link"][0]) == (link == 2)
    run_plan(rects, n)
    assert torch.equal(dst[:, 16:16 + 4096], win)
    assert bool((dst[:, :16] == GUARD).all()) and bool((dst[:, 16 + 4096:] == GUARD).all())
    fwin = base.view(torch.float32).view(R, P // 4)[r0:, 4:4 + 1024]
    want = fwin.to(torch.bfloat16)
    for start, vector in ((8, True), (1, False)):
        out = torch.full((rows, 1024 + 16), -3.0, dtype=torch.bfloat16, device="cuda")
        rects, n, fields, _ = compiled([(fwin, out[:, start:start + 1024])])
        assert int(fields["mode"][0]) == (MODE_F32_BF16_V8 if vector else 9)
        assert int(fields["src"][0]) - base.data_ptr() > 1 << 32
        run_plan(rects, n)
        assert_same_bits_or_nan(out[:, start:start + 1024], want)
        assert bool((out[:, :start] == -3.0).all()) and bool((out[:, start + 1024:] == -3.0).all())
    del base, win, fwin, want
    torch.cuda.empty_cache()

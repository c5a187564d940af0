"""Per-channel and per-tensor scaled FP8 pulls without a GPU: the numpy oracle pinned to torch CPU's
fixture, the torch rendering pinned to the oracle, and the native plan compiler
(tsb_scaled_fp8_compile_host) replayed on host memory against the oracle for FSDP -> TP reshards,
both kernel paths, replicated sources and MoE stacks."""

import os
import random
import time

import numpy as np
import pytest
import torch

from oracle.scaled_fp8_oracle import GRANULARITIES, bits_of, digest, fixture_inputs, quantize, replay, torch_quantize, widen
from tests.helpers import (HostBuffer, dest_scale_shape, expect_invalid, plan_windows, rand_full, region, shard_box,
                           shard_handles)
from torchstore_b200 import _native
from torchstore_b200.planner import StridedMem, build_rects

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "scaled_fp8_vectors.npz")
E4M3 = torch.float8_e4m3fn
CODE = {"channel": _native.TSB_SCALE_PER_CHANNEL, "tensor": _native.TSB_SCALE_PER_TENSOR}


def fixture_cases():
    """(name, granularity, dtype, x as exact float32, fp8 bytes or their sha256, scale_inv) per case and
    granularity; the inputs are rebuilt by scaled_fp8_oracle.fixture_inputs()."""
    d = np.load(GOLDEN)
    inputs = dict(fixture_inputs())
    out = []
    for i, name in enumerate(d["names"]):
        dtype = str(d[f"dtype{i}"])
        x = widen(bits_of(inputs[str(name)]), dtype)
        for g in GRANULARITIES:
            k = g[0]
            want_q = d[f"q_{k}{i}"] if f"q_{k}{i}" in d.files else str(d[f"q_sha_{k}{i}"])
            out.append((f"{name}-{g}", g, dtype, x, want_q, d[f"s_{k}{i}"]))
    return out


def test_fixture_inputs_are_the_recorded_ones():
    d = np.load(GOLDEN)
    inputs = dict(fixture_inputs())
    assert sorted(inputs) == sorted(map(str, d["names"]))
    for i, name in enumerate(d["names"]):
        x = inputs[str(name)]
        assert str(x.dtype).replace("torch.", "") == str(d[f"dtype{i}"]), name
        assert digest(bits_of(x)) == str(d[f"x_sha{i}"]), name


def finite_mask(s: np.ndarray, shape, granularity) -> np.ndarray:
    """Element mask of the groups whose scale is finite."""
    f = np.isfinite(s)
    if granularity == "tensor":
        f = f.reshape(f.shape + (1, 1))
    return np.broadcast_to(f, shape)


def assert_scaled_fp8_equal(q, s, want_q, want_s, granularity):
    """Bit-exact in finite groups; inside non-finite groups NaN-agnostic (a NaN byte is 0x7F or 0xFF
    depending on the platform that made it).  `want_q` is the fp8 bytes, or their sha256 for a case
    whose groups are all finite."""
    assert s.shape == want_s.shape
    assert np.array_equal(np.isfinite(s), np.isfinite(want_s))
    assert np.array_equal(s[np.isfinite(want_s)].view(np.uint32), want_s[np.isfinite(want_s)].view(np.uint32))
    assert np.array_equal(np.isnan(s), np.isnan(want_s))
    if isinstance(want_q, str):
        assert np.isfinite(want_s).all()
        assert digest(q) == want_q
        return
    fin = finite_mask(want_s, want_q.shape, granularity)
    assert np.array_equal(q[fin], want_q[fin])
    nan_q, nan_w = (q & 0x7F) == 0x7F, (want_q & 0x7F) == 0x7F
    assert np.array_equal(nan_q[~fin], nan_w[~fin])
    assert np.array_equal(q[~fin & ~nan_w], want_q[~fin & ~nan_w])


@pytest.mark.parametrize("case", fixture_cases(), ids=lambda c: c[0])
def test_oracle_matches_the_torch_cpu_fixture(case):
    _, g, _, x, want_q, want_s = case
    q, s = quantize(x, g)
    assert_scaled_fp8_equal(q, s, want_q, want_s, g)


def test_fixture_covers_the_special_groups():
    cases = {c[0]: c for c in fixture_cases()}
    for needle in ("zeros_subnormals_bfloat16", "zero_matrix_float16", "huge_bfloat16", "nonfinite_bfloat16",
                   "ragged_float32_129x257", "row_float16_1x16", "moe_bfloat16_3x130x260", "long_rows_bfloat16_3x16400",
                   "long_rows_float32_3x8200"):
        assert f"{needle}-channel" in cases and f"{needle}-tensor" in cases
    clamp = np.float32(np.float32(1e-4) / np.float32(448))
    assert (cases["zeros_subnormals_float32-channel"][5][:16] == clamp).all()  # zero and +-0 rows
    assert cases["zero_matrix_bfloat16-tensor"][5] == clamp
    s = cases["nonfinite_float32-channel"][5]
    assert s.shape == (130, 1) and np.isinf(s[5, 0]) and np.isnan(s[100, 0]) and np.isfinite(s).sum() == 128
    assert np.isnan(cases["nonfinite_float32-tensor"][5])  # one NaN poisons the whole matrix
    assert cases["moe_float32_3x130x260-tensor"][5].shape == (3,)


@pytest.mark.parametrize("case", [c for c in fixture_cases() if "nonfinite" not in c[0]], ids=lambda c: c[0])
def test_torch_rendering_matches_the_oracle_on_finite_data(case):
    _, g, dtype, x, _, _ = case
    q, s = torch_quantize(torch.from_numpy(x).to(getattr(torch, dtype)), g)
    want_q, want_s = quantize(x, g)
    assert np.array_equal(q.view(torch.uint8).numpy(), want_q)
    assert np.array_equal(s.numpy().view(np.uint32), want_s.view(np.uint32))


# ---- the plan compiler, replayed on host memory ----------------------------------------------------
def compile_pull(full, src_boxes, dst_box, g):
    """Plan (product planner, host memory) a pull of `full`'s `src_boxes` shards into the fp8
    destination `dst_box`; returns (dest, scale, (bands, pieces, tiles, n_groups), keepalive)."""
    handles, keep = shard_handles(full, src_boxes, lambda shard, off, loc: HostBuffer(shard, loc, shard.dtype))
    loc = dst_box[1]
    dest = torch.zeros(loc, dtype=E4M3)
    n, k = loc[-2:]
    scale = torch.zeros(dest_scale_shape(g, loc), dtype=torch.float32)
    _, pairs = plan_windows(handles, dest, dst_box)
    rects, nr = build_rects(pairs)
    targets = _native.make_sq_target_array(1)
    targets[0] = _native.SqTarget(dest.data_ptr(), scale.data_ptr(), dest.numel() // (n * k), n, k, CODE[g], 0)
    tables = _native.scaled_fp8_compile_host(0, rects, nr, targets, 1)
    return dest, scale, tables, (keep, rects, targets)


def check_tables(dest, tables, g):
    """Every destination element written exactly once; tiles sorted by group; one scale writer per group."""
    bands, pieces, tiles, n_groups = tables
    base = dest.data_ptr()
    hits = np.zeros(dest.numel(), dtype=np.int32)
    for b in bands:
        m = np.zeros((int(b["rows"]), int(b["cols"])), dtype=np.int32)
        for p in pieces[int(b["piece0"]): int(b["piece0"]) + int(b["n_pieces"])]:
            m[int(p["row0"]): int(p["row0"]) + int(p["rows"]), int(p["col0"]): int(p["col0"]) + int(p["cols"])] += 1
        assert (m == 1).all()
        o = int(b["dst"]) - base
        hits[o: o + m.size] += 1
    for t in tiles:
        for r in range(int(t["rows"])):
            o = int(t["dst"]) - base + r * int(t["pitch"])
            hits[o: o + int(t["cols"])] += 1
    assert (hits == 1).all()
    groups = tiles["group"].astype(np.int64)
    assert (np.diff(groups) >= 0).all() and (len(tiles) == 0 or groups.max() == n_groups - 1)
    writers = np.bincount(groups[tiles["scale_inv"] != 0], minlength=n_groups)
    assert (writers == 1).all()


def run_reshard(full, src_boxes, dst_box, g):
    dest, scale, tables, _keep = compile_pull(full, src_boxes, dst_box, g)
    check_tables(dest, tables, g)
    replay(*tables)
    want_q, want_s = quantize(region(full, *dst_box).float().numpy(), g)
    assert np.array_equal(dest.view(torch.uint8).numpy(), want_q)
    assert np.array_equal(scale.numpy().view(np.uint32), want_s.view(np.uint32))
    return tables


@pytest.mark.parametrize("g", GRANULARITIES)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("n,dst_dim", [(4, 0), (4, 1), (3, 1), (2, 0)])
def test_fsdp_rows_to_tp_reshard_replays_to_the_oracle(g, dtype, n, dst_dim):
    full = rand_full((300, 260), dtype, 10 * n + dst_dim)
    srcs = [shard_box(full.shape, n, r, 0) for r in range(n)]  # row boundaries at 75/150/225 or 100/200
    for d in range(n):
        bands, pieces, tiles, _ = run_reshard(full, srcs, shard_box(full.shape, n, d, dst_dim), g)
        if g == "channel":
            assert len(tiles) == 0 and len(bands) > 0  # 260 columns fit the stage
        else:
            assert len(bands) == 0 and len(tiles) > 0


@pytest.mark.parametrize("dtype,cols", [(torch.bfloat16, 16400), (torch.float32, 8200), (torch.float32, 8192)])
def test_long_rows_take_the_two_pass_path(dtype, cols):
    """Rows past the 32 KiB stage: one group per row, read by tiles; 8192 f32 (exactly 32 KiB) is staged."""
    full = rand_full((6, cols), dtype, 11)
    srcs = [shard_box(full.shape, 3, r, 1) for r in range(3)]  # column shards at unaligned boundaries
    bands, _, tiles, n_groups = run_reshard(full, srcs, ((0, 0), (6, cols)), "channel")
    if cols * full.element_size() > 32768:
        assert len(bands) == 0 and n_groups == 6 and len(tiles) >= 18
    else:
        assert len(tiles) == 0 and len(bands) == 6


def test_per_tensor_over_shards_and_tiles():
    full = rand_full((700, 300), torch.bfloat16, 12)  # 210 000 elements: several 16384-element tiles per shard
    srcs = [shard_box(full.shape, 3, r, 0) for r in range(3)]
    _, _, tiles, n_groups = run_reshard(full, srcs, ((0, 0), (700, 300)), "tensor")
    assert n_groups == 1 and len(tiles) > 3


def test_exact_match_whole_tensor():
    full = rand_full((129, 257), torch.bfloat16, 3)
    bands, pieces, _, _ = run_reshard(full, [((0, 0), (129, 257))], ((0, 0), (129, 257)), "channel")
    assert sum(int(b["rows"]) for b in bands) == 129 and len(pieces) == len(bands)


@pytest.mark.parametrize("g", GRANULARITIES)
def test_replicated_sources_are_read_once(g):
    full = rand_full((256, 200), torch.bfloat16, 4)
    srcs = [shard_box(full.shape, 2, r % 2, 0) for r in range(4)]  # (Replicate, Shard(0)): every shard twice
    dest, _, tables, _keep = compile_pull(full, srcs, shard_box(full.shape, 2, 1, 1), g)
    check_tables(dest, tables, g)
    run_reshard(full, srcs, shard_box(full.shape, 2, 1, 1), g)


@pytest.mark.parametrize("g", GRANULARITIES)
@pytest.mark.parametrize("dst_dim", [1, 2])
def test_moe_stack(g, dst_dim):
    full = rand_full((3, 130, 260), torch.float32, 5)
    srcs = [shard_box(full.shape, 3, r, 1) for r in range(3)]
    for d in range(2):
        run_reshard(full, srcs, shard_box(full.shape, 2, d, dst_dim), g)
    _, _, _, n_groups = run_reshard(full, [((0, 0, 0), (3, 130, 260))], ((0, 0, 0), (3, 130, 260)), g)
    assert n_groups == (3 if g == "tensor" else 0)


def test_random_reshards():
    rng = random.Random(7)
    for i in range(16):
        shape = (rng.randint(1, 400), rng.randint(1, 400))
        n_src, n_dst = rng.randint(1, 5), rng.randint(1, 4)
        sd, dd = rng.randint(0, 1), rng.randint(0, 1)
        full = rand_full(shape, rng.choice([torch.bfloat16, torch.float16, torch.float32]), i)
        srcs = [shard_box(shape, n_src, r, sd) for r in range(n_src)]
        for d in range(n_dst):
            dst = shard_box(shape, n_dst, d, dd)
            if 0 not in dst[1]:
                run_reshard(full, srcs, dst, GRANULARITIES[i % 2])


@pytest.mark.parametrize("g", GRANULARITIES)
def test_uncovered_and_twice_covered_groups_fail(g):
    full = rand_full((300, 260), torch.bfloat16, 6)
    srcs = [shard_box(full.shape, 4, r, 0) for r in range(4)]
    msg = expect_invalid(lambda: compile_pull(full, srcs[:3], ((0, 0), (300, 260)), g))  # rows 225.. missing
    assert ("target 0 group (0, 225)" if g == "channel" else "target 0 group (0)") in msg
    # overlapping shards: rows 100..150 twice (not a dedupable replica: different boxes)
    expect_invalid(lambda: compile_pull(full, [((0, 0), (150, 260)), ((100, 0), (200, 260))], ((0, 0), (300, 260)), g))
    # columns: one shard missing, and two overlapping
    cs = [shard_box(full.shape, 3, r, 1) for r in range(3)]
    expect_invalid(lambda: compile_pull(full, cs[:2], ((0, 0), (300, 260)), g))
    expect_invalid(lambda: compile_pull(full, [((0, 0), (300, 200)), ((0, 100), (300, 160))], ((0, 0), (300, 260)), g))


def test_mixed_dtype_groups_fail():
    a = torch.zeros(64, 64, dtype=torch.bfloat16)
    b = torch.zeros(64, 64, dtype=torch.float32)
    dst = torch.zeros(64, 128, dtype=E4M3)
    for g, shape in (("channel", (64, 1)), ("tensor", ())):
        scale = torch.zeros(shape)
        pairs = [(StridedMem.from_tensor(a), StridedMem.from_tensor(dst[:, :64])),
                 (StridedMem.from_tensor(b), StridedMem.from_tensor(dst[:, 64:]))]
        rects, n = build_rects(pairs)
        targets = _native.make_sq_target_array(1)
        targets[0] = _native.SqTarget(dst.data_ptr(), scale.data_ptr(), 1, 64, 128, CODE[g], 0)
        msg = expect_invalid(lambda: _native.scaled_fp8_compile_host(0, rects, n, targets, 1))
        assert "different dtypes" in msg and "target 0 group (0" in msg
    # different dtypes in different rows are fine per channel (each row is one group) and not per tensor
    top, bottom = torch.zeros(32, 128, dtype=torch.bfloat16), torch.zeros(32, 128, dtype=torch.float32)
    pairs = [(StridedMem.from_tensor(top), StridedMem.from_tensor(dst[:32])),
             (StridedMem.from_tensor(bottom), StridedMem.from_tensor(dst[32:]))]
    rects, n = build_rects(pairs)
    for g, shape, ok in (("channel", (64, 1), True), ("tensor", (), False)):
        scale = torch.zeros(shape)
        targets = _native.make_sq_target_array(1)
        targets[0] = _native.SqTarget(dst.data_ptr(), scale.data_ptr(), 1, 64, 128, CODE[g], 0)
        if ok:
            bands, _, _, _ = _native.scaled_fp8_compile_host(0, rects, n, targets, 1)
            assert sorted(set(bands["src_dtype"].tolist())) == [5, 6]
        else:
            expect_invalid(lambda: _native.scaled_fp8_compile_host(0, rects, n, targets, 1))


def test_bad_targets_and_granularity_codes_fail():
    src = torch.zeros(64, 64, dtype=torch.bfloat16)
    dst = torch.zeros(64, 64, dtype=E4M3)
    scale = torch.zeros(64, 1)
    rects, n = build_rects([(StridedMem.from_tensor(src), StridedMem.from_tensor(dst))])

    def compile_with(**kw):
        t = dict(dst=dst.data_ptr(), scale_inv=scale.data_ptr(), batch=1, rows=64, cols=64,
                 granularity=_native.TSB_SCALE_PER_CHANNEL, pad=0)
        t.update(kw)
        targets = _native.make_sq_target_array(1)
        targets[0] = _native.SqTarget(**t)
        return _native.scaled_fp8_compile_host(0, rects, n, targets, 1)

    bands, pieces, tiles, _ = compile_with()
    assert len(bands) == 1 and int(pieces[0]["vec"]) == 1 and len(tiles) == 0
    for kw in (dict(dst=0), dict(scale_inv=0), dict(rows=0), dict(cols=0), dict(batch=0), dict(scale_inv=scale.data_ptr() + 2),
               dict(dst=dst.data_ptr() + 4096), dict(pad=1)):  # dst + 4096: the rect lies in no target
        expect_invalid(lambda: compile_with(**kw))
    for code in (0, 3, 0xFFFFFFFF):
        msg = expect_invalid(lambda: compile_with(granularity=code))
        assert "granularity" in msg
    with pytest.raises(_native.TsbError) as e:  # a bf16 destination is not scaled fp8
        r2, n2 = build_rects([(StridedMem.from_tensor(src), StridedMem.from_tensor(src))])
        targets = _native.make_sq_target_array(1)
        targets[0] = _native.SqTarget(src.data_ptr(), scale.data_ptr(), 1, 64, 64, _native.TSB_SCALE_PER_CHANNEL, 0)
        _native.scaled_fp8_compile_host(0, r2, n2, targets, 1)
    assert e.value.code == _native.TSB_ERR_UNSUPPORTED


@pytest.mark.parametrize("g", GRANULARITIES)
def test_full_size_llama3_8b_targets_compile_in_time_of_pieces_not_elements(g):
    """Llama-3-8B w1 [14336, 4096] pulled from 8 FSDP row shards (a per-tensor group of 58.7 M elements),
    compiled from addresses alone: no memory behind them is touched."""
    rows, cols, n_src = 14336, 4096, 8
    src_base, dst_base, scale_base = 1 << 40, 1 << 41, 1 << 42
    pairs = []
    for r in range(n_src):
        r0, r1 = r * rows // n_src, (r + 1) * rows // n_src
        src = StridedMem(src_base + r * (1 << 30), (r1 - r0, cols), (cols, 1), torch.bfloat16, 0)
        dst = StridedMem(dst_base + r0 * cols, (r1 - r0, cols), (cols, 1), E4M3, 0)
        pairs.append((src, dst))
    rects, n = build_rects(pairs)
    targets = _native.make_sq_target_array(1)
    targets[0] = _native.SqTarget(dst_base, scale_base, 1, rows, cols, CODE[g], 0)
    t0 = time.perf_counter()
    bands, pieces, tiles, n_groups = _native.scaled_fp8_compile_host(0, rects, n, targets, 1)
    elapsed = time.perf_counter() - t0
    assert elapsed < 2.0, elapsed
    if g == "tensor":
        assert n_groups == 1 and len(tiles) == rows * cols // 16384 and len(bands) == 0
    else:
        assert len(bands) == rows // 4 and len(tiles) == 0  # 8 KiB bf16 rows: four per 32 KiB stage

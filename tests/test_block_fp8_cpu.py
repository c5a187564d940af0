"""Block-scaled FP8 pulls without a GPU: the numpy oracle pinned to torch CPU's fixture, the torch
rendering pinned to the oracle, and the native plan compiler (tsb_block_fp8_compile_host) replayed on
host memory against the oracle for FSDP -> TP reshards, replicated sources and MoE stacks."""

import os
import random

import numpy as np
import pytest
import torch

from oracle.block_fp8_oracle import bits_of, digest, fixture_inputs, quantize, replay, torch_quantize, widen
from tests.helpers import HostBuffer, expect_invalid, plan_windows, rand_full, region, shard_box, shard_handles
from torchstore_b200 import _native
from torchstore_b200.planner import StridedMem, build_rects

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "block_fp8_vectors.npz")
E4M3 = torch.float8_e4m3fn
B = 128


def fixture_cases():
    """(name, dtype, x as exact float32, fp8 bytes or their sha256, scale_inv) of every fixture case;
    the inputs are rebuilt by block_fp8_oracle.fixture_inputs()."""
    d = np.load(GOLDEN)
    inputs = dict(fixture_inputs())
    out = []
    for i, name in enumerate(d["names"]):
        dtype = str(d[f"dtype{i}"])
        x = widen(bits_of(inputs[str(name)]), dtype)
        want_q = d[f"q{i}"] if f"q{i}" in d.files else str(d[f"q_sha{i}"])
        out.append((str(name), dtype, x, want_q, d[f"s{i}"]))
    return out


def test_fixture_inputs_are_the_recorded_ones():
    d = np.load(GOLDEN)
    inputs = dict(fixture_inputs())
    assert sorted(inputs) == sorted(map(str, d["names"]))
    for i, name in enumerate(d["names"]):
        x = inputs[str(name)]
        assert str(x.dtype).replace("torch.", "") == str(d[f"dtype{i}"]), name
        assert digest(bits_of(x)) == str(d[f"x_sha{i}"]), name


def finite_block_mask(s: np.ndarray, shape) -> np.ndarray:
    """Element mask of the blocks whose scale is finite."""
    *_, n, k = shape
    return np.repeat(np.repeat(np.isfinite(s), B, axis=-2), B, axis=-1)[..., :n, :k]


def assert_block_fp8_equal(q, s, want_q, want_s):
    """Bit-exact in finite blocks; inside non-finite blocks NaN-agnostic (a NaN byte is 0x7F or 0xFF
    depending on the platform that made it).  `want_q` is the fp8 bytes, or their sha256 for a case
    whose blocks are all finite."""
    assert np.array_equal(np.isfinite(s), np.isfinite(want_s))
    assert np.array_equal(s[np.isfinite(want_s)].view(np.uint32), want_s[np.isfinite(want_s)].view(np.uint32))
    assert np.array_equal(np.isnan(s), np.isnan(want_s))
    if isinstance(want_q, str):
        assert np.isfinite(want_s).all()
        assert digest(q) == want_q
        return
    fin = finite_block_mask(want_s, want_q.shape)
    assert np.array_equal(q[fin], want_q[fin])
    nan_q, nan_w = (q & 0x7F) == 0x7F, (want_q & 0x7F) == 0x7F
    assert np.array_equal(nan_q[~fin], nan_w[~fin])
    assert np.array_equal(q[~fin & ~nan_w], want_q[~fin & ~nan_w])


@pytest.mark.parametrize("case", fixture_cases(), ids=lambda c: c[0])
def test_oracle_matches_the_torch_cpu_fixture(case):
    _, _, x, want_q, want_s = case
    q, s = quantize(x)
    assert_block_fp8_equal(q, s, want_q, want_s)


def test_fixture_covers_the_special_blocks():
    names = [c[0] for c in fixture_cases()]
    for needle in ("zeros_subnormals_bfloat16", "huge_bfloat16", "nonfinite_bfloat16", "ragged_float32_129x257",
                   "row_float16_1x16", "moe_bfloat16_3x130x260"):
        assert needle in names
    s = {c[0]: c[4] for c in fixture_cases()}
    assert s["zeros_subnormals_float32"][0, 0] == np.float32(np.float32(1e-4) / np.float32(448))  # the clamp
    assert np.isinf(s["nonfinite_float32"]).sum() == 1 and np.isnan(s["nonfinite_float32"]).sum() == 1


def test_scalar_division_in_torch_is_not_the_formula():
    """``448.0 / amax`` in torch is reciprocal-then-multiply; on the fixture it differs from the
    oracle's correctly rounded division somewhere."""
    differs = 0
    for _, _, x, _, _ in fixture_cases():
        xf = torch.from_numpy(np.abs(x))
        *lead, n, k = xf.shape
        nb, kb = -(-n // B), -(-k // B)
        pad = torch.nn.functional.pad(xf, (0, kb * B - k, 0, nb * B - n))
        amax = torch.maximum(pad.reshape(*lead, nb, B, kb, B).amax(dim=(-3, -1)), torch.tensor(1e-4))
        true_scale = (np.float32(448) / amax.numpy()).astype(np.float32)
        rdiv = (448.0 / amax).numpy()
        fin = np.isfinite(true_scale)
        differs += int((rdiv[fin].view(np.uint32) != true_scale[fin].view(np.uint32)).sum())
    assert differs > 0


@pytest.mark.parametrize("case", [c for c in fixture_cases() if "nonfinite" not in c[0]], ids=lambda c: c[0])
def test_torch_rendering_matches_the_oracle_on_finite_data(case):
    _, dtype, x, _, _ = case
    q, s = torch_quantize(torch.from_numpy(x).to(getattr(torch, dtype)))
    want_q, want_s = quantize(x)
    assert np.array_equal(q.view(torch.uint8).numpy(), want_q)
    assert np.array_equal(s.numpy().view(np.uint32), want_s.view(np.uint32))


# ---- the plan compiler, replayed on host memory ----------------------------------------------------
def compile_pull(full, src_boxes, dst_box):
    """Plan (product planner, host memory) a pull of `full`'s `src_boxes` shards into the fp8
    destination `dst_box`; returns (dest, scale, blocks, pieces, keepalive)."""
    handles, keep = shard_handles(full, src_boxes, lambda shard, off, loc: HostBuffer(shard, loc, shard.dtype))
    loc = dst_box[1]
    dest = torch.zeros(loc, dtype=E4M3)
    *lead, n, k = loc
    scale = torch.zeros(*lead, -(-n // B), -(-k // B), dtype=torch.float32)
    _, pairs = plan_windows(handles, dest, dst_box)
    rects, nr = build_rects(pairs)
    targets = _native.make_target_array(1)
    targets[0] = _native.BqTarget(dest.data_ptr(), scale.data_ptr(), dest.numel() // (n * k), n, k)
    blocks, pieces = _native.block_fp8_compile_host(0, rects, nr, targets, 1)
    return dest, scale, blocks, pieces, (keep, rects, targets)


def check_tiling(blocks, pieces):
    for blk in blocks:
        m = np.zeros((int(blk["rows"]), int(blk["cols"])), dtype=np.int32)
        for p in pieces[int(blk["piece0"]): int(blk["piece0"]) + int(blk["n_pieces"])]:
            m[int(p["row0"]): int(p["row0"]) + int(p["rows"]), int(p["col0"]): int(p["col0"]) + int(p["cols"])] += 1
        assert (m == 1).all()


def run_reshard(full, src_boxes, dst_box):
    dest, scale, blocks, pieces, _keep = compile_pull(full, src_boxes, dst_box)
    check_tiling(blocks, pieces)
    replay(blocks, pieces)
    want_q, want_s = quantize(region(full, *dst_box).float().numpy())
    assert np.array_equal(dest.view(torch.uint8).numpy(), want_q)
    assert np.array_equal(scale.numpy().view(np.uint32), want_s.view(np.uint32))
    return blocks, pieces


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("n,dst_dim", [(4, 0), (4, 1), (3, 1), (2, 0)])
def test_fsdp_rows_to_tp_reshard_replays_to_the_oracle(dtype, n, dst_dim):
    full = rand_full((300, 260), dtype, 10 * n + dst_dim)
    srcs = [shard_box(full.shape, n, r, 0) for r in range(n)]  # boundaries at 75/150/225 or 100/200: not multiples of 128
    straddled = False
    for d in range(n):
        blocks, pieces = run_reshard(full, srcs, shard_box(full.shape, n, d, dst_dim))
        straddled |= len(pieces) > len(blocks)
    assert straddled == (dst_dim == 1)  # column shards hold every row: some block spans two source shards


def test_exact_match_whole_tensor():
    full = rand_full((129, 257), torch.bfloat16, 3)
    blocks, pieces = run_reshard(full, [((0, 0), (129, 257))], ((0, 0), (129, 257)))
    assert len(blocks) == 6 and len(pieces) == 6


def test_replicated_sources_are_read_once():
    full = rand_full((256, 200), torch.bfloat16, 4)
    srcs = [shard_box(full.shape, 2, r % 2, 0) for r in range(4)]  # (Replicate, Shard(0)): every shard twice
    blocks, pieces = run_reshard(full, srcs, shard_box(full.shape, 2, 1, 1))
    check_tiling(blocks, pieces)


@pytest.mark.parametrize("dst_dim", [1, 2])
def test_moe_stack(dst_dim):
    full = rand_full((3, 130, 260), torch.float32, 5)
    srcs = [shard_box(full.shape, 3, r, 1) for r in range(3)]
    for d in range(2):
        run_reshard(full, srcs, shard_box(full.shape, 2, d, dst_dim))
    run_reshard(full, [((0, 0, 0), (3, 130, 260))], ((0, 0, 0), (3, 130, 260)))


def test_random_reshards():
    rng = random.Random(7)
    for i in range(12):
        shape = (rng.randint(1, 400), rng.randint(1, 400))
        n_src, n_dst = rng.randint(1, 5), rng.randint(1, 4)
        sd, dd = rng.randint(0, 1), rng.randint(0, 1)
        full = rand_full(shape, rng.choice([torch.bfloat16, torch.float16, torch.float32]), i)
        srcs = [shard_box(shape, n_src, r, sd) for r in range(n_src)]
        for d in range(n_dst):
            dst = shard_box(shape, n_dst, d, dd)
            if 0 not in dst[1]:
                run_reshard(full, srcs, dst)


def test_uncovered_and_twice_covered_blocks_fail():
    full = rand_full((300, 260), torch.bfloat16, 6)
    srcs = [shard_box(full.shape, 4, r, 0) for r in range(4)]
    msg = expect_invalid(lambda: compile_pull(full, srcs[:3], ((0, 0), (300, 260))))  # rows 225.. missing
    assert "target 0 block (0, 1" in msg
    # overlapping shards: rows 0..150 twice (not a dedupable replica: different boxes)
    expect_invalid(lambda: compile_pull(full, [((0, 0), (150, 260)), ((100, 0), (200, 260))], ((0, 0), (300, 260))))


def test_bad_targets_fail():
    src = torch.zeros(64, 64, dtype=torch.bfloat16)
    dst = torch.zeros(64, 64, dtype=E4M3)
    scale = torch.zeros(1, 1)
    rects, n = build_rects([(StridedMem.from_tensor(src), StridedMem.from_tensor(dst))])

    def compile_with(**kw):
        t = dict(dst=dst.data_ptr(), scale_inv=scale.data_ptr(), batch=1, rows=64, cols=64)
        t.update(kw)
        targets = _native.make_target_array(1)
        targets[0] = _native.BqTarget(**t)
        return _native.block_fp8_compile_host(0, rects, n, targets, 1)

    blocks, pieces = compile_with()
    assert len(blocks) == 1 and int(pieces[0]["vec"]) == 1
    for kw in (dict(dst=0), dict(scale_inv=0), dict(rows=0), dict(cols=0), dict(batch=0), dict(scale_inv=scale.data_ptr() + 2),
               dict(dst=dst.data_ptr() + 4096)):  # the last one: the rect lies in no target
        expect_invalid(lambda: compile_with(**kw))
    with pytest.raises(_native.TsbError) as e:  # a bf16 destination is not block-scaled fp8
        r2, n2 = build_rects([(StridedMem.from_tensor(src), StridedMem.from_tensor(src))])
        targets = _native.make_target_array(1)
        targets[0] = _native.BqTarget(src.data_ptr(), scale.data_ptr(), 1, 64, 64)
        _native.block_fp8_compile_host(0, r2, n2, targets, 1)
    assert e.value.code == _native.TSB_ERR_UNSUPPORTED

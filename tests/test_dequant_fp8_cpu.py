"""Dequantising pulls without a GPU: the numpy oracle pinned to torch CPU's fixture, the native plan
compiler (tsb_dequant_fp8_compile_host) replayed on host memory against the oracle for FSDP -> TP
reshards with unaligned shard offsets, replicated sources and MoE stacks, and the validation of
register(), pull() and the compiler."""

import os
import random
import time
import types

import numpy as np
import pytest
import torch

from oracle.dequant_fp8_oracle import (DST, GRANULARITIES, SCALE_SET, decode_e4m3, dequantize, digest, fixture_inputs,
                                       replay, scale_shape, torch_dequantize)
from tests.helpers import cuda_like, expect_invalid, no_export, plan_windows, region, shard_box, shard_handles
from torchstore_b200 import _native
from torchstore_b200.direct_weight_sync import (DirectWeightSyncDest, DirectWeightSyncSource, RDMAWeightHandle,
                                                source_scale_shapes)
from torchstore_b200.planner import StridedMem, build_rects
from torchstore_b200.transport.types import TensorSlice

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "dequant_fp8_vectors.npz")
E4M3 = torch.float8_e4m3fn
CODE = {"block": _native.TSB_SCALE_PER_BLOCK, "channel": _native.TSB_SCALE_PER_CHANNEL,
        "tensor": _native.TSB_SCALE_PER_TENSOR}


def torch_bits(y: torch.Tensor) -> np.ndarray:
    return y.view(torch.int16 if y.element_size() == 2 else torch.int32).numpy().view(
        np.uint16 if y.element_size() == 2 else np.uint32)


def is_nan_bits(bits: np.ndarray, dst: str) -> np.ndarray:
    if dst == "float32":
        return np.isnan(bits.view(np.float32))
    if dst == "float16":
        return np.isnan(bits.view(np.float16))
    return (bits & 0x7FFF) > 0x7F80


# ---- the oracle against the torch CPU fixture ------------------------------------------------------
def test_fixture_inputs_are_the_recorded_ones():
    d = np.load(GOLDEN)
    inputs = fixture_inputs()
    assert [n for n, *_ in inputs] == list(map(str, d["names"]))
    for i, (name, g, r0, c0, q, s) in enumerate(inputs):
        assert str(d[f"g{i}"]) == g and list(d[f"off{i}"]) == [r0, c0], name
        assert digest(q.view(torch.uint8).numpy()) == str(d[f"q_sha{i}"]), name
        assert digest(s.numpy().view(np.uint32)) == str(d[f"s_sha{i}"]), name


@pytest.mark.parametrize("dst", list(DST))
@pytest.mark.parametrize("i", range(len(fixture_inputs())))
def test_oracle_matches_the_torch_cpu_fixture(i, dst):
    d = np.load(GOLDEN)
    name, g, r0, c0, q, s = fixture_inputs()[i]
    got = dequantize(q.view(torch.uint8).numpy(), s.numpy(), g, r0, c0, dst)
    if f"y_{dst}{i}" in d.files:  # NaN bits are platform-specific: NaN-agnostic there, bit-exact elsewhere
        want = d[f"y_{dst}{i}"]
        nan = is_nan_bits(want, dst)
        assert np.array_equal(is_nan_bits(got, dst), nan)
        assert np.array_equal(got[~nan], want[~nan])
    else:
        assert digest(got) == str(d[f"y_sha_{dst}{i}"]), name


def test_all_bytes_table_covers_the_special_products():
    d = np.load(GOLDEN)
    i = list(map(str, d["names"])).index("all_bytes")
    x = decode_e4m3(np.arange(256, dtype=np.uint8))
    assert np.isnan(x[0x7F]) and np.isnan(x[0xFF]) and x[0x7E] == 448 and x[1] == 2.0 ** -9
    bf16 = d[f"y_bfloat16{i}"].reshape(len(SCALE_SET), 256)
    f16 = d[f"y_float16{i}"].reshape(len(SCALE_SET), 256)
    f32 = d[f"y_float32{i}"].reshape(len(SCALE_SET), 256).view(np.float32)
    row = {float(s): k for k, s in enumerate(SCALE_SET) if np.isfinite(s)}
    k = row[float(np.float32(2.0 ** -140))]
    assert 0 < f32[k, 1] < np.finfo(np.float32).tiny  # an f32-subnormal product, not flushed
    assert f16[row[1000.0], 0x7E] == 0x7C00 and bf16[row[float(np.float32(7.589e35))], 0x7E] == 0x7F80  # overflow to Inf
    assert (f32[row[0.0], :0x7F] == 0).all() and f32[row[-0.5], 0x38] == -0.5


def test_torch_rendering_matches_the_oracle():
    for name, g, r0, c0, q, s in fixture_inputs()[1:]:
        for dst, dtype in DST.items():
            want = dequantize(q.view(torch.uint8).numpy(), s.numpy(), g, r0, c0, dst)
            assert np.array_equal(torch_bits(torch_dequantize(q, s, g, r0, c0, dtype)), want), (name, dst)


# ---- the plan compiler, replayed on host memory ----------------------------------------------------
def global_scale(g, shape, seed):
    """A global scale tensor of the full tensor (anchored at the origin)."""
    gen = torch.Generator().manual_seed(seed)
    return torch.rand(scale_shape(g, shape), generator=gen) * 0.01 + 1e-4


def local_scale(full_scale, g, off, loc):
    """The groups a shard at `off` of shape `loc` touches (checkpoint semantics)."""
    *lead_off, r0, c0 = off
    *lead, n, k = loc
    lead_idx = tuple(slice(o, o + e) for o, e in zip(lead_off, lead))
    if g == "block":
        return full_scale[lead_idx + (slice(r0 // 128, -(-(r0 + n) // 128)), slice(c0 // 128, -(-(c0 + k) // 128)))].contiguous()
    if g == "channel":
        return full_scale[lead_idx + (slice(r0, r0 + n),)].contiguous()
    return full_scale[lead_idx].contiguous()


class FakeScaledBuffer:
    """Host-memory stand-in for ScaledNvlinkBuffer (the planner only reads these attributes)."""

    def __init__(self, shard, scale, g, r0, c0):
        self.shard, self.scale, self.granularity, self.row0, self.col0 = shard, scale, g, r0, c0


def compile_pull(q_full, full_scale, g, src_boxes, dst_box, dst_dtype):
    """Plan a pull of `q_full`'s shards (each with its own slice of the global scale) into a `dst_dtype`
    window `dst_box`; returns (dest, tiles, keepalive)."""
    handles, keep = shard_handles(q_full, src_boxes, lambda shard, off, loc: FakeScaledBuffer(
        shard, local_scale(full_scale, g, off, loc), g, off[-2], off[-1]))
    dest = torch.zeros(dst_box[1], dtype=dst_dtype)
    ops, pairs = plan_windows(handles, dest, dst_box)
    sources, index = [], {}
    for op in ops:
        buf = op.rdma_buffer
        if id(buf) not in index:
            index[id(buf)] = len(sources)
            n, k = buf.shard.shape[-2:]
            sources.append(_native.DqSource(buf.shard.data_ptr(), buf.scale.data_ptr(), buf.shard.numel() // (n * k), n, k,
                                            buf.row0, buf.col0, CODE[g], 0))
    rects, nr = build_rects(pairs, dequantise=True)  # TSB_I8 rects for int8 sources
    arr = _native.make_dq_source_array(max(1, len(sources)))
    for i, s in enumerate(sources):
        arr[i] = s
    tiles = _native.dequant_fp8_compile_host(0, rects, nr, arr, len(sources))
    return dest, tiles, (keep, rects, arr, handles)


def run_reshard(q_full, full_scale, g, src_boxes, dst_box, dst_dtype):
    dest, tiles, _keep = compile_pull(q_full, full_scale, g, src_boxes, dst_box, dst_dtype)
    assert all(int(t["rows"]) * int(t["cols"]) <= 16384 and int(t["rows"]) <= 256 for t in tiles)
    replay(tiles)
    dst = str(dst_dtype).replace("torch.", "")
    want = dequantize(region(q_full, *dst_box).view(torch.uint8).numpy(), region_scale(full_scale, g, dst_box),
                      g, dst_box[0][-2], dst_box[0][-1], dst)
    assert np.array_equal(torch_bits(dest), want)
    return tiles


def region_scale(full_scale, g, box):
    return local_scale(full_scale, g, *box).numpy()


def fp8_full(shape, seed):
    gen = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=gen) * 4).to(E4M3)


@pytest.mark.parametrize("g", GRANULARITIES)
@pytest.mark.parametrize("dst_dtype", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("n,dst_dim", [(6, 0), (6, 1), (3, 1), (4, 0)])
def test_fsdp_rows_to_tp_reshard_replays_to_the_oracle(g, dst_dtype, n, dst_dim):
    """FSDP(n) row shards starting mid-block (300 rows over 6: 50-row shards) into column- and row-parallel
    TP destinations."""
    q = fp8_full((300, 260), 10 * n + dst_dim)
    s = global_scale(g, q.shape, n)
    srcs = [shard_box(q.shape, n, r, 0) for r in range(n)]
    for d in range(2):
        run_reshard(q, s, g, srcs, shard_box(q.shape, 2, d, dst_dim), dst_dtype)


@pytest.mark.parametrize("g", GRANULARITIES)
def test_replicated_sources_are_read_once(g):
    q = fp8_full((256, 200), 4)
    s = global_scale(g, q.shape, 4)
    srcs = [shard_box(q.shape, 2, r % 2, 0) for r in range(4)]  # (Replicate, Shard(0)): every shard twice
    tiles = run_reshard(q, s, g, srcs, ((0, 0), (256, 200)), torch.bfloat16)
    assert sum(int(t["rows"]) * int(t["cols"]) for t in tiles) == 256 * 200


@pytest.mark.parametrize("g", GRANULARITIES)
@pytest.mark.parametrize("dst_dtype", [torch.bfloat16, torch.float16, torch.float32])
def test_ep_sharded_moe_stack(g, dst_dtype):
    q = fp8_full((4, 130, 260), 5)
    s = global_scale(g, q.shape, 5)
    experts = [shard_box(q.shape, 2, r, 0) for r in range(2)]  # EP: experts 0-1 and 2-3
    run_reshard(q, s, g, experts, ((0, 0, 0), (4, 130, 260)), dst_dtype)
    rows = [shard_box(q.shape, 3, r, 1) for r in range(3)]  # rows cut at 44 / 88, mid-block
    for d in range(2):
        run_reshard(q, s, g, rows, shard_box(q.shape, 2, d, 2), dst_dtype)


def test_block_pieces_follow_the_global_block_grid():
    """A shard at row 50 carries blocks 0..2 of rows 50..300; its tiles break at global rows 128 and 256."""
    q = fp8_full((300, 260), 8)
    s = global_scale("block", q.shape, 8)
    tiles = run_reshard(q, s, "block", [((0, 0), (50, 260)), ((50, 0), (250, 260))], ((0, 0), (300, 260)), torch.bfloat16)
    assert sorted({int(t["rows"]) for t in tiles}) == [44, 50, 78, 128]  # 0..50 | 50..128, 128..256, 256..300
    assert all(int(t["cols"]) <= 128 for t in tiles)
    assert (tiles["scale_step"] == 0).all()


def test_random_reshards():
    rng = random.Random(7)
    for i in range(12):
        shape = (rng.randint(1, 400), rng.randint(1, 400))
        n_src, n_dst = rng.randint(1, 5), rng.randint(1, 4)
        sd, dd = rng.randint(0, 1), rng.randint(0, 1)
        g = GRANULARITIES[i % 3]
        q = fp8_full(shape, i)
        s = global_scale(g, shape, i)
        srcs = [shard_box(shape, n_src, r, sd) for r in range(n_src)]
        for d in range(n_dst):
            dst = shard_box(shape, n_dst, d, dd)
            if 0 not in dst[1]:
                run_reshard(q, s, g, srcs, dst, rng.choice([torch.bfloat16, torch.float16, torch.float32]))


@pytest.mark.parametrize("g", GRANULARITIES)
def test_full_size_llama3_8b_compile(g):
    """Llama-3-8B w1 [14336, 4096] from 6 FSDP row shards (boundaries mid-block) into bf16, compiled from
    addresses alone: no memory behind them is touched."""
    rows, cols, n_src = 14336, 4096, 6
    src_base, dst_base, scale_base = 1 << 40, 1 << 41, 1 << 42
    pairs, sources = [], _native.make_dq_source_array(n_src)
    for r in range(n_src):
        r0, r1 = r * rows // n_src, (r + 1) * rows // n_src
        src = StridedMem(src_base + r * (1 << 30), (r1 - r0, cols), (cols, 1), E4M3, 0)
        dst = StridedMem(dst_base + 2 * r0 * cols, (r1 - r0, cols), (cols, 1), torch.bfloat16, 0)
        pairs.append((src, dst))
        sources[r] = _native.DqSource(src.ptr, scale_base + r * (1 << 20), 1, r1 - r0, cols, r0, 0, CODE[g], 0)
    rects, n = build_rects(pairs)
    t0 = time.perf_counter()
    tiles = _native.dequant_fp8_compile_host(0, rects, n, sources, n_src)
    assert time.perf_counter() - t0 < 2.0
    assert int((tiles["rows"].astype(np.int64) * tiles["cols"]).sum()) == rows * cols
    assert (tiles["vec"] == 1).all()
    if g == "block":
        assert len(tiles) == sum(len(range(r * rows // n_src // 128, -(-((r + 1) * rows // n_src) // 128))) for r in range(n_src)) * 32
    else:
        assert len(tiles) == sum(-(-((r + 1) * rows // n_src - r * rows // n_src) // 4) for r in range(n_src))  # 4 rows each


# ---- compiler errors ------------------------------------------------------------------------------
def test_compile_errors_name_the_rect_or_source():
    q = torch.zeros(64, 64, dtype=E4M3)
    s = torch.zeros(64, 1)
    dst = torch.zeros(64, 64, dtype=torch.bfloat16)

    def compile_with(src_t=q, dst_t=dst, **kw):
        f = dict(src=q.data_ptr(), scale=s.data_ptr(), batch=1, rows=64, cols=64, row0=0, col0=0,
                 granularity=_native.TSB_SCALE_PER_CHANNEL, pad=0)
        f.update(kw)
        arr = _native.make_dq_source_array(1)
        arr[0] = _native.DqSource(**f)
        rects, n = build_rects([(StridedMem.from_tensor(src_t), StridedMem.from_tensor(dst_t))])
        return _native.dequant_fp8_compile_host(0, rects, n, arr, 1)

    assert len(compile_with()) == 1
    assert "rect 0" in expect_invalid(lambda: compile_with(src=q.data_ptr() + 8192))  # the rect's source lies in no source
    for kw in (dict(scale=0), dict(rows=0), dict(scale=s.data_ptr() + 2), dict(pad=1), dict(granularity=0)):
        assert "source 0" in expect_invalid(lambda: compile_with(**kw))
    bf = torch.zeros(64, 64, dtype=torch.bfloat16)  # source not float8_e4m3fn
    assert "float8_e4m3fn" in expect_invalid(lambda: compile_with(src_t=bf, dst_t=torch.zeros(64, 64, dtype=torch.float32),
                                                                  src=bf.data_ptr()))
    f64 = torch.zeros(64, 64, dtype=torch.float64)  # destination not f32/bf16/f16
    with pytest.raises((_native.TsbError, NotImplementedError)):
        compile_with(dst_t=f64)
    arr = _native.make_dq_source_array(1)
    arr[0] = _native.DqSource(q.data_ptr(), s.data_ptr(), 1, 64, 64, 0, 0, _native.TSB_SCALE_PER_CHANNEL, 0)
    rects, n = build_rects([(StridedMem.from_tensor(q), StridedMem.from_tensor(dst))])
    rects[0].dst_dtype = _native.TSB_F8E5M2  # an fp8 destination: not dequantised
    assert "f32, bf16 or f16" in expect_invalid(lambda: _native.dequant_fp8_compile_host(0, rects, n, arr, 1))
    wide = torch.zeros(64, 128, dtype=E4M3)  # strided source rows: not a box of a [64, 64] source
    arr = _native.make_dq_source_array(1)
    arr[0] = _native.DqSource(wide.data_ptr(), s.data_ptr(), 1, 64, 64, 0, 0, _native.TSB_SCALE_PER_CHANNEL, 0)
    rects, n = build_rects([(StridedMem.from_tensor(wide[:, :64]), StridedMem.from_tensor(dst))])
    assert "rect 0" in expect_invalid(lambda: _native.dequant_fp8_compile_host(0, rects, n, arr, 1))


# ---- register / pull validation (before anything is exported or launched) ---------------------------
no_export = pytest.fixture(no_export)


def test_register_errors_raise_before_export(no_export):
    w = torch.zeros(256, 256, dtype=E4M3)
    src = DirectWeightSyncSource()
    with pytest.raises(ValueError, match="not in the state dict"):
        src.register({"w": w}, 0, block_scales={"x": torch.zeros(2, 2)})
    with pytest.raises(ValueError, match="more than one"):
        src.register({"w": w}, 0, block_scales={"w": torch.zeros(2, 2)}, tensor_scales={"w": torch.zeros(())})
    with pytest.raises(ValueError, match="transfer_dtype"):
        src.register({"w": w}, 0, transfer_dtype=torch.bfloat16, channel_scales={"w": torch.zeros(256, 1)})
    with pytest.raises(TypeError, match="float8_e4m3fn"):
        src.register({"w": w.to(torch.bfloat16)}, 0, block_scales={"w": torch.zeros(2, 2)})
    for bad in (torch.zeros(256, dtype=E4M3), torch.zeros(0, 4, dtype=E4M3), torch.zeros(4, 8, dtype=E4M3).t(), w):
        with pytest.raises(ValueError, match="non-empty contiguous CUDA"):  # 1-D, empty, strided, and on the CPU
            src.register({"w": bad}, 0, tensor_scales={"w": torch.zeros(())})
    assert src._handles == {}


def test_scale_shapes_are_anchored_at_the_global_origin():
    # 7168 rows over 6 ranks: rank 1 holds rows 1195..2389, which touch blocks 9..18 (10 block rows)
    assert source_scale_shapes("block", (1195, 7168), 1195, 0) == [(10, 56)]
    assert source_scale_shapes("block", (128, 128), 0, 0) == [(1, 1)]
    assert source_scale_shapes("block", (3, 100, 300), 100, 5) == [(3, 2, 3)]
    assert source_scale_shapes("channel", (3, 100, 300), 100, 5) == [(3, 100, 1)]
    assert source_scale_shapes("tensor", (3, 100, 300), 0, 0) == [(3,), (3, 1)]


def test_pull_errors_raise_before_compile(no_export):
    def handles(kinds):
        return [RDMAWeightHandle(rdma_buffer=types.SimpleNamespace(granularity=k, dtype=E4M3), source_rank=r,
                                 tensor_slice=TensorSlice((0, 0), (r,), (8, 8), (8, 8), (2,))) for r, k in enumerate(kinds)]

    dest = {"w": torch.zeros(8, 8, dtype=torch.bfloat16)}
    check = DirectWeightSyncDest._check_dequant
    with pytest.raises(ValueError, match="mix scaled fp8 and unscaled"):
        check({"w": handles(["block", None])}, dest, set())
    with pytest.raises(ValueError, match="granularities"):
        check({"w": handles(["block", "channel"])}, dest, set())
    with pytest.raises(TypeError, match="bfloat16, float16, float32"):
        check({"w": handles(["tensor"])}, {"w": torch.zeros(8, 8, dtype=torch.int32)}, set())
    with pytest.raises(TypeError, match="bfloat16, float16, float32"):
        check({"w": handles(["tensor"])}, {"w": torch.zeros(8, 8, dtype=torch.float8_e5m2)}, set())
    with pytest.raises(ValueError, match="contiguous with at least 2 dims"):
        check({"w": handles(["tensor"])}, {"w": torch.zeros(64, dtype=torch.bfloat16)}, set())
    with pytest.raises(ValueError, match="contiguous with at least 2 dims"):
        check({"w": handles(["tensor"])}, {"w": torch.zeros(8, 8, dtype=torch.bfloat16).t()}, set())
    assert check({"w": handles(["block", "block"])}, dest, set()) == {"w"}
    assert check({"w": handles(["block"])}, {"w": torch.zeros(8, 8, dtype=E4M3)}, set()) == set()  # byte move
    assert check({"w": handles([None])}, dest, set()) == set()
    # the same errors through pull(): raised before any plan is compiled
    import asyncio

    with pytest.raises(ValueError, match="mix"):
        asyncio.run(DirectWeightSyncDest().pull({"w": handles(["block", None])}, dest))
    # a scaled destination fed by scaled fp8 handles keeps the quantising path's TypeError (no requantising)
    with pytest.raises(TypeError, match="bf16, f16 or f32 handles"):
        DirectWeightSyncDest._check_scales({"w": handles(["block"])}, {"w": cuda_like(torch.zeros(8, 8, dtype=E4M3))},
                                           {"block_scales": {"w": torch.zeros(1, 1)}})


def test_store_path_refuses_scales():
    import asyncio

    from torchstore_b200 import state_dict_utils

    for kw in ("block_scales", "channel_scales", "tensor_scales"):
        with pytest.raises(NotImplementedError):
            asyncio.run(state_dict_utils.put_state_dict(None, {"w": torch.zeros(1)}, "k", direct_rdma=False,
                                                        **{kw: {"w": torch.zeros(1)}}))


def test_dequantising_names_never_take_the_all_gather(monkeypatch):
    """_try_all_gather votes no when the published shard is fp8 and the destination bf16."""
    import torch.distributed as dist

    from torchstore_b200 import collectives, state_dict_utils

    votes = []
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda: 2)
    monkeypatch.setattr(dist, "get_rank", lambda: 0)
    monkeypatch.setattr(dist, "all_reduce", lambda t, op=None: votes.append(int(t.item())))
    monkeypatch.setattr(collectives, "is_allgather_shaped", lambda *a: True)
    monkeypatch.setattr(collectives, "all_gather_state_dict", lambda *a: pytest.fail("all-gather taken"))
    shard = torch.zeros(4, 8, dtype=E4M3)
    ts = TensorSlice((0, 0), (0,), (8, 8), (4, 8), (2,))
    buf = types.SimpleNamespace(_keepalive=shard, granularity="block")
    cache = types.SimpleNamespace(sources={"k": types.SimpleNamespace(_handles={"w": RDMAWeightHandle(buf, ts, 0)})},
                                  registered={"k"})
    assert not state_dict_utils._try_all_gather(cache, "k", {"w": torch.zeros(8, 8, dtype=torch.bfloat16)})
    assert votes == [0]

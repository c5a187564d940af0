"""Source-side quantisation without a GPU: the numpy oracle pinned to torch CPU's fixture, the native compiler
(tsb_source_quant_compile_host) replayed on host memory against the oracle, its tables checked to cover every
element exactly once under the right shard-local group, a full-size compile, and every validation error of
``DirectWeightSyncSource.register(quantize=...)``."""

import os
import time

import numpy as np
import pytest
import torch

from oracle.source_quant_oracle import (GRANULARITIES, bits_of, digest, element_scales, fixture_inputs, quantize, replay,
                                        synth_f32, torch_quantize, widen)
from torchstore_b200 import _native
from torchstore_b200.direct_weight_sync import DirectWeightSyncSource, source_scale_shapes
from torchstore_b200.transport.types import TensorSlice

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "source_quant_vectors.npz")
CODE = {"block": _native.TSB_SCALE_PER_BLOCK, "channel": _native.TSB_SCALE_PER_CHANNEL, "tensor": _native.TSB_SCALE_PER_TENSOR}
DT = {"bfloat16": _native.TSB_BF16, "float16": _native.TSB_F16, "float32": _native.TSB_F32}


def fixture_cases():
    """(name, x as exact float32, granularity, row0, col0, fp8 bytes or their sha256, scale_inv) per case."""
    d = np.load(GOLDEN)
    inputs = {name: (x, g, r0, c0) for name, x, g, r0, c0 in fixture_inputs()}
    out = []
    for i, name in enumerate(d["names"]):
        x, g, r0, c0 = inputs[str(name)]
        want_q = d[f"q{i}"] if f"q{i}" in d.files else str(d[f"q_sha{i}"])
        out.append((str(name), widen(bits_of(x), str(d[f"dtype{i}"])), g, r0, c0, want_q, d[f"s{i}"]))
    return out


def assert_source_quant_equal(q, s, want_q, want_s, g, r0, c0):
    """Bit-exact in finite groups; inside non-finite groups NaN-agnostic (a NaN byte is 0x7F or 0xFF depending
    on the platform that made it).  `want_q` is the fp8 bytes, or their sha256 when every group is finite."""
    assert s.shape == want_s.shape
    fin_s = np.isfinite(want_s)
    assert np.array_equal(np.isfinite(s), fin_s) and np.array_equal(np.isnan(s), np.isnan(want_s))
    assert np.array_equal(s[fin_s].view(np.uint32), want_s[fin_s].view(np.uint32))
    if isinstance(want_q, str):
        assert fin_s.all()
        assert digest(q) == want_q
        return
    fin = np.isfinite(element_scales(want_s, g, want_q.shape, r0, c0))
    assert np.array_equal(q[fin], want_q[fin])
    nan_q, nan_w = (q & 0x7F) == 0x7F, (want_q & 0x7F) == 0x7F
    assert np.array_equal(nan_q[~fin], nan_w[~fin])
    assert np.array_equal(q[~fin & ~nan_w], want_q[~fin & ~nan_w])


def test_fixture_inputs_are_the_recorded_ones():
    d = np.load(GOLDEN)
    inputs = {name: (x, g, r0, c0) for name, x, g, r0, c0 in fixture_inputs()}
    assert sorted(inputs) == sorted(map(str, d["names"]))
    for i, name in enumerate(d["names"]):
        x, g, r0, c0 = inputs[str(name)]
        assert str(x.dtype).replace("torch.", "") == str(d[f"dtype{i}"]), name
        assert list(d[f"where{i}"]) == [g, str(r0), str(c0)], name
        assert digest(bits_of(x)) == str(d[f"x_sha{i}"]), name


@pytest.mark.parametrize("case", fixture_cases(), ids=lambda c: c[0])
def test_oracle_matches_the_torch_cpu_fixture(case):
    _, x, g, r0, c0, want_q, want_s = case
    q, s = quantize(x, g, r0, c0)
    assert s.shape == source_scale_shapes(g, x.shape, r0, c0)[0]
    assert_source_quant_equal(q, s, want_q, want_s, g, r0, c0)


def test_fixture_covers_the_special_groups():
    cases = {c[0]: c for c in fixture_cases()}
    for g in GRANULARITIES:
        for dtype in ("bfloat16", "float16", "float32"):
            for where in ("0_0", "37_70", "128_256"):
                assert f"{g}_{dtype}_300x200_at_{where}" in cases
            assert f"{g}_{dtype}_moe_3x130x260_at_100_5" in cases
            _, x, _, r0, c0, want_q, s = cases[f"{g}_{dtype}_special_at_37_70"]
            assert np.isnan(s).any() and not isinstance(want_q, str)
            if g != "tensor":
                assert np.isinf(s).any() or g == "block"  # an Inf amax: scale_inv Inf per channel
                assert (s == np.float32(1e-4) / np.float32(448)).any()  # the all-zero group / the 1e-4 clamp


def test_full_tensor_equivalence_at_group_aligned_boundaries():
    """Shards cut on group boundaries: the concatenated bytes and scales equal quantising the full tensor."""
    x = widen(bits_of(synth_f32((512, 384), 77).to(torch.bfloat16)), "bfloat16")
    for g in ("block", "channel"):
        full_q, full_s = quantize(x, g)
        parts = [quantize(x[r0:r0 + 128], g, r0, 0) for r0 in range(0, 512, 128)]
        assert np.array_equal(np.concatenate([q for q, _ in parts]), full_q)
        assert np.array_equal(np.concatenate([s for _, s in parts]).view(np.uint32), full_s.view(np.uint32))


# ---------------------------------------------------------------------------------------------
# compiled tables replayed on host memory
# ---------------------------------------------------------------------------------------------
def host_shard(x: torch.Tensor, g: str, r0: int, c0: int, misalign: int = 0):
    """Host buffers of one target: source bits (optionally starting `misalign` elements into a larger array,
    so its address is not 16-byte aligned), fp8 and scale outputs, and the SourceQuantTarget over them."""
    bits = bits_of(x)
    backing = np.zeros(bits.size + misalign + 8, dtype=bits.dtype)
    backing[misalign: misalign + bits.size] = bits.reshape(-1)
    src = backing[misalign: misalign + bits.size]
    q = np.full(x.shape, 0xAB, dtype=np.uint8)
    s = np.full(source_scale_shapes(g, tuple(x.shape), r0, c0)[0], np.nan, dtype=np.float32)
    rows, cols = x.shape[-2:]
    t = _native.SourceQuantTarget(src.ctypes.data, q.ctypes.data, s.ctypes.data, x.numel() // (rows * cols), rows, cols,
                                  r0, c0, DT[str(x.dtype).replace("torch.", "")], CODE[g])
    return backing, q, s, t


def compile_host(targets, flags=0):
    arr = _native.make_source_quant_target_array(max(1, len(targets)))
    for i, t in enumerate(targets):
        arr[i] = t
    return _native.source_quant_compile_host(0, arr, len(targets), flags)


def coverage(units, tiles, t, es):
    """Per element of target t: how many units/tiles write it, and the scale_inv index each one uses."""
    n = t.batch * t.rows * t.cols
    count = np.zeros(n, dtype=np.int64)
    group = np.full(n, -1, dtype=np.int64)
    for u in units:
        if not (t.src <= int(u["src"]) < t.src + n * es):
            continue
        first = (int(u["src"]) - t.src) // es
        assert int(u["dst"]) - t.dst == first and int(u["src_pitch"]) == t.cols * es and int(u["dst_pitch"]) == t.cols
        s0 = (int(u["scale_inv"]) - t.scale_inv) // 4
        for r in range(int(u["rows"])):
            idx = first + r * t.cols + np.arange(int(u["cols"]))
            count[idx] += 1
            group[idx] = s0 + (r if int(u["per_row"]) else 0)
    writer = {int(x["group"]): (int(x["scale_inv"]) - t.scale_inv) // 4 for x in tiles if int(x["scale_inv"])}
    for x in tiles:
        if not (t.src <= int(x["src"]) < t.src + n * es):
            continue
        first = (int(x["src"]) - t.src) // es
        assert int(x["dst"]) - t.dst == first and int(x["rows"]) == 1
        idx = first + np.arange(int(x["cols"]))
        count[idx] += 1
        group[idx] = writer[int(x["group"])]
    return count, group


CASES = [(g, dtype, shape, r0, c0, mis)
         for g in GRANULARITIES
         for dtype in (torch.bfloat16, torch.float16, torch.float32)
         for shape, r0, c0, mis in (((300, 200), 0, 0, 0), ((300, 200), 37, 70, 0), ((256, 384), 128, 256, 0),
                                    ((3, 130, 260), 100, 5, 0), ((129, 257), 37, 70, 1), ((2, 9000), 5, 0, 0),
                                    ((1, 16), 127, 127, 0))]


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"{c[0]}-{str(c[1])[6:]}-{'x'.join(map(str, c[2]))}-at{c[3]}_{c[4]}-mis{c[5]}")
def test_replayed_tables_match_the_oracle_and_cover_each_element_once(case):
    g, dtype, shape, r0, c0, mis = case
    x = synth_f32(shape, 31 + len(shape) + r0 + c0).to(dtype)
    backing, q, s, t = host_shard(x, g, r0, c0, mis)
    units, tiles, n_groups = compile_host([t])
    es = x.element_size()
    count, group = coverage(units, tiles, t, es)
    assert (count == 1).all()
    want_group = np.arange(s.size).reshape(s.shape)
    assert np.array_equal(group, element_scales(want_group, g, shape, r0, c0).reshape(-1))
    if mis:
        assert not units["vec"].any() and not tiles["vec"].any()
    replay(units, tiles, n_groups)
    want_q, want_s = quantize(widen(bits_of(x), str(dtype)[6:]), g, r0, c0)
    assert np.array_equal(q, want_q)
    assert np.array_equal(s.view(np.uint32), want_s.view(np.uint32))
    del backing


def test_paths_and_unit_shapes():
    """Blocks and short per-channel rows are staged units; per-tensor groups and rows over 32 KiB are two-pass
    tiles; the first partial block row and column of an unaligned shard are units with fewer rows / columns."""
    x = synth_f32((300, 200), 5).to(torch.bfloat16)
    _, _, _, t = host_shard(x, "block", 37, 70)
    units, tiles, ng = compile_host([t])
    assert len(tiles) == 0 and ng == 0 and not units["per_row"].any()
    assert sorted(set(units["rows"].tolist())) == [81, 91, 128] and sorted(set(units["cols"].tolist())) == [14, 58, 128]
    _, _, _, t = host_shard(x, "channel", 0, 0)
    units, tiles, ng = compile_host([t])
    assert len(tiles) == 0 and units["per_row"].all() and units["rows"].sum() == 300
    _, _, _, t = host_shard(x, "tensor", 0, 0)
    units, tiles, ng = compile_host([t])
    assert len(units) == 0 and ng == 1 and (tiles["scale_inv"] != 0).sum() == 1
    long = synth_f32((2, 16400), 6).to(torch.bfloat16)
    _, _, _, t = host_shard(long, "channel", 0, 0)
    units, tiles, ng = compile_host([t])
    assert len(units) == 0 and ng == 2 and len(tiles) == 4


def test_units_fit_one_cta_and_are_grouped_by_dtype():
    """A unit holds at most 4 * 256 16-element chunks (one per thread and register slot of the kernel), and units come
    grouped bf16, f16, f32 (one launch per dtype), whatever the order of the targets."""
    targets, keep = [], []
    for dtype, shape in ((torch.float32, (64, 300)), (torch.bfloat16, (300, 273)), (torch.float16, (40, 1000)),
                         (torch.bfloat16, (256, 384))):
        for g in ("block", "channel"):
            backing, q, s, t = host_shard(synth_f32(shape, 9).to(dtype), g, 37, 0)
            targets.append(t)
            keep += [backing, q, s]
    units, _, _ = compile_host(targets)
    chunks = units["rows"].astype(np.int64) * ((units["cols"].astype(np.int64) + 15) // 16)
    assert chunks.max() <= 1024
    order = [{_native.TSB_BF16: 0, _native.TSB_F16: 1, _native.TSB_F32: 2}[int(d)] for d in units["src_dtype"]]
    assert order == sorted(order) and set(order) == {0, 1, 2}


def test_full_size_llama3_8b_fsdp8_compile_is_quick():
    """Every linear weight of Llama-3-8B (32 layers), cut into 8 FSDP row shards, compiled per granularity."""
    shapes = {"wq": (4096, 4096), "wk": (1024, 4096), "wv": (1024, 4096), "wo": (4096, 4096), "w1": (14336, 4096),
              "w2": (4096, 14336), "w3": (14336, 4096)}
    base = 1 << 40
    for g in GRANULARITIES:
        targets = []
        addr = base
        for _layer in range(32):
            for n, k in shapes.values():
                for r in range(8):
                    rows = n // 8
                    targets.append(_native.SourceQuantTarget(addr, addr + (1 << 38), addr + (1 << 39), 1, rows, k,
                                                             r * rows, 0, _native.TSB_BF16, CODE[g]))
                    addr += rows * k * 2 + 4096
        t0 = time.perf_counter()
        units, tiles, _ = compile_host(targets)
        took = time.perf_counter() - t0
        assert took < 10.0, (g, took)
        n_elem = sum(t.rows * t.cols for t in targets)
        assert int((units["rows"].astype(np.int64) * units["cols"]).sum()) + int(tiles["cols"].astype(np.int64).sum()) == n_elem


def test_native_refuses_bad_targets():
    x = synth_f32((4, 16), 1).to(torch.bfloat16)
    _, _, _, t = host_shard(x, "block", 0, 0)
    for field, value, needle in (("src_dtype", _native.TSB_F8E4M3, "src_dtype"), ("granularity", 7, "granularity"),
                                 ("rows", 0, "empty"), ("scale_inv", 0, "NULL"), ("src", t.src + 1, "aligned"),
                                 ("scale_inv", t.scale_inv + 2, "4-byte")):
        bad = _native.SourceQuantTarget.from_buffer_copy(t)
        setattr(bad, field, value)
        with pytest.raises(_native.TsbError, match=needle) as e:
            compile_host([t, bad])
        assert e.value.code == _native.TSB_ERR_INVALID and "target 1" in str(e.value)


# ---------------------------------------------------------------------------------------------
# register() validation: raises before anything is exported or allocated
# ---------------------------------------------------------------------------------------------
@pytest.fixture
def nothing_exported(monkeypatch):
    from torchstore_b200 import direct_weight_sync as dws

    def boom(*a, **k):
        raise AssertionError("exported or compiled before validation finished")

    monkeypatch.setattr(dws.HbmDescriptor, "from_tensor", staticmethod(boom))
    monkeypatch.setattr(dws.Plans, "build_source_quant", classmethod(boom))
    monkeypatch.setattr(dws.Plans, "build", classmethod(boom))


def _w(*shape, dtype=torch.bfloat16):
    return torch.zeros(*shape, dtype=dtype)


@pytest.mark.parametrize("sd, quant, scales, exc, needle", [
    ({"w": _w(4, 4)}, {"v": "block"}, {}, ValueError, "not in the state dict"),
    ({"w": _w(4, 4)}, {"w": "row"}, {}, ValueError, "must be one of"),
    ({"w": _w(4, 4), "f": _w(4, 4, dtype=torch.float8_e4m3fn)}, {"f": "block"},
     {"block_scales": {"f": torch.zeros(1, 1)}}, ValueError, "in quantize and in one of"),
    ({"w": _w(4, 4, dtype=torch.int32)}, {"w": "block"}, {}, TypeError, "bfloat16, float16 or float32"),
    ({"w": _w(4, 4, dtype=torch.float64)}, {"w": "tensor"}, {}, TypeError, "bfloat16, float16 or float32"),
    ({"w": _w(0, 4)}, {"w": "channel"}, {}, ValueError, "is empty"),
    ({"w": _w(16)}, {"w": "channel"}, {}, ValueError, "needs at least 2 dims"),
    ({"w": _w(8, 8)[:, ::2]}, {"w": "block"}, {}, ValueError, "is not contiguous"),
    ({"w": _w(8, 8)}, {"w": "block"}, {}, ValueError, "must live on a CUDA device, not cpu"),
], ids=["unknown-name", "unknown-granularity", "also-scaled", "int32", "float64", "empty", "1-d", "strided", "host"])
def test_register_validation(nothing_exported, sd, quant, scales, exc, needle):
    src = DirectWeightSyncSource()
    with pytest.raises(exc, match=needle):
        src.register(sd, rank=0, quantize=quant, **scales)
    assert src._handles == {} and src._quantized == {} and not src._quant_plans


def test_register_validation_with_tensor_slices(nothing_exported):
    ts = TensorSlice((4, 0), (1,), (8, 4), (4, 4), (2,))
    with pytest.raises(ValueError, match="must live on a CUDA device"):
        DirectWeightSyncSource().register({"w": _w(4, 4)}, rank=1, tensor_slices={"w": ts}, quantize={"w": "block"})


def test_store_path_refuses_quantize():
    import asyncio

    from torchstore_b200 import state_dict_utils

    with pytest.raises(NotImplementedError, match="quantize needs direct_rdma=True"):
        asyncio.run(state_dict_utils.put_state_dict(None, {"w": _w(4, 4)}, "k", quantize={"w": "block"}))

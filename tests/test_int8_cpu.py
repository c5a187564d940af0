"""Scaled INT8 destinations without a GPU: the numpy oracle pinned to torch CPU's fixture, the compiled block / band /
tile tables of TSB_I8 rects (byte-identical to the float8_e4m3fn tables) replayed on host memory against the
oracle, the C-ABI's refusals around TSB_I8, and the Python routing and refusals of int8 names in direct weight
sync, raised before anything is compiled."""

import asyncio
import os
import types

import numpy as np
import pytest
import torch

from oracle.int8_oracle import (GRANULARITIES, SPECIALS, bits_of, digest, fixture_inputs, quantize, replay_block,
                                replay_scaled, same_scales, scales_of_amax, synth_f32, torch_quantize, widen)
from tests.helpers import Boom, fake_dest, no_export, scaled_handle
from torchstore_b200 import _native
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest
from torchstore_b200.planner import StridedMem, build_rects

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "int8_vectors.npz")
E4M3 = torch.float8_e4m3fn
CODE = {"channel": _native.TSB_SCALE_PER_CHANNEL, "tensor": _native.TSB_SCALE_PER_TENSOR}
KW = {"block": "block_scales", "channel": "channel_scales", "tensor": "tensor_scales"}


def u32(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


# ---- the formula -------------------------------------------------------------------------------------------------
def test_scale_step_edge_cases():
    amax = np.array([0, 1e-5, 127, 254, np.finfo(np.float32).max, np.inf, np.nan], dtype=np.float32)
    scale, scale_inv = scales_of_amax(amax)
    assert scale[0] == np.float32(127) / np.float32(1e-4) and scale_inv[0] == np.float32(1e-4) / np.float32(127)
    assert scale[1] == scale[0]  # the floor
    assert scale[2] == 1 and scale_inv[2] == 1 and scale[3] == 0.5
    assert scale[5] == 0 and np.isinf(scale_inv[5])
    assert np.isnan(scale[6]) and np.isnan(scale_inv[6])


def test_ties_round_half_to_even_and_non_finite_groups_give_zero():
    x = np.array([[127, 0.5, 1.5, 2.5, -0.5, -1.5, -2.5, 126.5, -126.5]], dtype=np.float32)
    q, s = quantize(x, "channel")
    assert q.tolist() == [[127, 0, 2, 2, 0, -2, -2, 126, -126]] and s[0, 0] == 1
    for bad in (np.nan, np.inf, -np.inf):
        q, s = quantize(np.array([[1.0, bad, -3.0]], dtype=np.float32), "channel")
        assert (q == 0).all() and (np.isnan(s).all() if np.isnan(bad) else np.isinf(s).all())


def test_finite_groups_never_saturate():
    for spread in (0, 8, 60):
        x = synth_f32((64, 300), 31 + spread, spread=spread).numpy()
        for g in GRANULARITIES:
            q, _ = quantize(x, g)
            assert q.min() >= -127 and q.max() <= 127


# ---- the fixture -------------------------------------------------------------------------------------------------
def test_fixture_inputs_are_the_recorded_ones():
    d = np.load(GOLDEN)
    cases = fixture_inputs()
    assert [c[0] for c in cases] == [str(n) for n in d["names"]]
    for i, (name, x, g) in enumerate(cases):
        assert str(x.dtype).replace("torch.", "") == str(d[f"dtype{i}"]) and str(d[f"granularity{i}"]) == g, name
        assert digest(bits_of(x)) == str(d[f"x_sha{i}"]), name


def test_fixture_covers_every_regime():
    names = {c[0] for c in fixture_inputs()}
    for g in GRANULARITIES:
        for dtype in ("bfloat16", "float16", "float32"):
            assert {f"{g}_{dtype}_300x200", f"{g}_{dtype}_moe_3x130x260", f"{g}_{dtype}_special_7x130x260"} <= names
    assert SPECIALS == ("ties", "zero", "nan", "inf", "nan_inf", "max", "subnormal")


@pytest.mark.parametrize("i", range(27))
def test_oracle_matches_the_torch_cpu_fixture(i):
    d = np.load(GOLDEN)
    name, x, g = fixture_inputs()[i]
    q, s = quantize(widen(bits_of(x), str(x.dtype)[6:]), g)
    assert digest(q.view(np.uint8)) == str(d[f"q_sha{i}"]), name
    assert same_scales(s, d[f"s{i}"]), name
    if "special" in name:  # NaN and Inf groups: q = 0 and scale_inv NaN / Inf
        for k, kind in enumerate(SPECIALS):
            if kind in ("nan", "inf", "nan_inf"):
                assert (q[k] == 0).all(), (name, kind)
                assert (np.isnan(s[k]) if kind != "inf" else np.isinf(s[k])).all(), (name, kind)
            if kind == "ties":
                assert (s[k] == 1).all() and (q[k] % 2 == 0).any()


def test_torch_rendering_matches_the_oracle_on_odd_shapes():
    for g in GRANULARITIES:
        for shape in ((1, 1), (129, 3), (2, 5, 257)):
            x = synth_f32(shape, 5)
            q, s = quantize(x.numpy(), g)
            tq, ts = torch_quantize(x, g)
            assert np.array_equal(q, tq.numpy()) and same_scales(s, ts.numpy())


# ---- the C-ABI ---------------------------------------------------------------------------------------------------
def host_pull(full: torch.Tensor, cuts, dest_dtype):
    """Row shards of a host tensor pulled into one whole-tensor destination: (dest, rects, n, keep)."""
    dest = torch.full(full.shape, 0x55, dtype=torch.uint8).view(dest_dtype)
    shards = [full[a:b].contiguous() for a, b in cuts]
    d = StridedMem.from_tensor(dest)
    pairs = [(StridedMem.from_tensor(s), d.sub((slice(a, b), slice(None)))) for s, (a, b) in zip(shards, cuts)]
    rects, n = build_rects(pairs, quantise=True)
    return dest, rects, n, shards


def block_case(dest_dtype, dtype=torch.bfloat16):
    full = synth_f32((300, 260), 11).to(dtype)
    dest, rects, n, keep = host_pull(full, ((0, 150), (150, 300)), dest_dtype)
    scale = torch.full((3, 3), -1.0)
    tg = _native.make_target_array(1)
    tg[0] = _native.BqTarget(dest.data_ptr(), scale.data_ptr(), 1, 300, 260)
    compile_ = lambda f=0: _native.block_fp8_compile_host(0, rects, n, tg, 1, f)  # noqa: E731
    return full, "block", dest, scale, rects, n, compile_, (keep, tg)


def scaled_case(g, cols, dest_dtype, dtype=torch.bfloat16):
    full = synth_f32((40, cols), 12).to(dtype)
    dest, rects, n, keep = host_pull(full, ((0, 13), (13, 40)), dest_dtype)
    scale = torch.full((40, 1) if g == "channel" else (), -1.0)
    tg = _native.make_sq_target_array(1)
    tg[0] = _native.SqTarget(dest.data_ptr(), scale.data_ptr(), 1, 40, cols, CODE[g], 0)
    compile_ = lambda f=0: _native.scaled_fp8_compile_host(0, rects, n, tg, 1, f)  # noqa: E731
    return full, g, dest, scale, rects, n, compile_, (keep, tg)


REGIMES = (("block", None), ("channel", 260), ("channel", 16400), ("tensor", 260))  # 16400: two-pass rows


def case(g, cols, dest_dtype, dtype=torch.bfloat16):
    return block_case(dest_dtype, dtype) if g == "block" else scaled_case(g, cols, dest_dtype, dtype)


def test_rect_filler_emits_tsb_i8_only_for_quantising_windows():
    assert _native.TSB_I8 == 10 and _native.dtype_code(torch.int8) == _native.TSB_U8
    for dtype in (torch.bfloat16, torch.float16, torch.float32):
        _, _, _, _, rects, n, _, _ = block_case(torch.int8, dtype)
        assert n == 2 and all(rects[i].dst_dtype == _native.TSB_I8 for i in range(n))
        assert rects[0].src_dtype == _native.cast_code(dtype)
    src, dst = torch.zeros(4, 4, dtype=torch.bfloat16), torch.zeros(4, 4, dtype=torch.int8)
    with pytest.raises(NotImplementedError, match="no fused cast kernel"):
        build_rects([(StridedMem.from_tensor(src), StridedMem.from_tensor(dst))])
    i8 = torch.zeros(4, 4, dtype=torch.int8)
    rects, n = build_rects([(StridedMem.from_tensor(i8), StridedMem.from_tensor(dst))], quantise=True)
    assert rects[0].src_dtype == rects[0].dst_dtype == _native.TSB_U8  # int8 -> int8 stays a byte move


def same_tables(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        if isinstance(x, np.ndarray):
            assert x.dtype == y.dtype and x.tobytes() == y.tobytes()
        else:
            assert x == y


@pytest.mark.parametrize("g,cols", REGIMES)
def test_int8_tables_are_the_fp8_tables(g, cols):
    """The destination dtype selects kernels, not tables: TSB_I8 rects compile to the bytes of TSB_F8E4M3 rects
    over the same buffers."""
    *_, rects, n, compile_, _keep = case(g, cols, torch.int8)
    assert all(rects[i].dst_dtype == _native.TSB_I8 for i in range(n))
    i8 = compile_()
    for i in range(n):  # the same buffers, the rects relabelled float8_e4m3fn
        rects[i].dst_dtype = _native.TSB_F8E4M3
    same_tables(compile_(), i8)


@pytest.mark.parametrize("dtype", (torch.bfloat16, torch.float16, torch.float32), ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("g,cols", REGIMES)
def test_replayed_tables_match_the_oracle(g, cols, dtype):
    full, g, dest, scale, rects, n, compile_, _keep = case(g, cols, torch.int8, dtype)
    tables = compile_()
    if g == "block":
        replay_block(*tables)
    else:
        bands, pieces, tiles, n_groups = tables
        assert (len(tiles) > 0) == (cols == 16400 or g == "tensor")
        replay_scaled(*tables)
    want_q, want_s = quantize(widen(bits_of(full), str(dtype)[6:]), g)
    assert np.array_equal(dest.numpy(), want_q)
    assert np.array_equal(u32(scale.numpy()).reshape(-1), u32(want_s).reshape(-1))


def expect(code, fn, needle):
    with pytest.raises(_native.TsbError, match=needle) as e:
        fn()
    assert e.value.code == code


@pytest.mark.parametrize("g,cols", REGIMES)
def test_c_refusals(g, cols):
    *_, rects, n, compile_, keep = case(g, cols, torch.int8)
    # TSB_I8 with the power-of-two scale flag
    expect(_native.TSB_ERR_INVALID, lambda: compile_(_native.TSB_QUANT_UE8M0), "TSB_QUANT_UE8M0")
    # one plan writes one destination dtype
    rects[1].dst_dtype = _native.TSB_F8E4M3
    expect(_native.TSB_ERR_INVALID, compile_, "one destination dtype")
    rects[0].dst_dtype, rects[1].dst_dtype = _native.TSB_F8E4M3, _native.TSB_I8
    expect(_native.TSB_ERR_INVALID, compile_, "one destination dtype")
    # other destination codes stay refused
    for bad in (_native.TSB_U8, _native.TSB_F8E5M2, 11):
        rects[0].dst_dtype = rects[1].dst_dtype = bad
        expect(_native.TSB_ERR_UNSUPPORTED, compile_, "float8_e4m3fn or int8")
    rects[0].dst_dtype = rects[1].dst_dtype = _native.TSB_I8
    compile_()


def test_tsb_i8_stays_out_of_the_copy_plan_and_the_other_kinds():
    lib = _native.lib()
    for other in (_native.TSB_F32, _native.TSB_BF16, _native.TSB_U8, _native.TSB_I8, _native.TSB_F8E4M3):
        assert lib.tsb_cast_supported(other, _native.TSB_I8) == 0 and lib.tsb_cast_supported(_native.TSB_I8, other) == 0
    src, dst = torch.zeros(8, 16, dtype=torch.bfloat16), torch.zeros(8, 16, dtype=torch.int8)
    rects, n = build_rects([(StridedMem.from_tensor(src), StridedMem.from_tensor(dst))], quantise=True)
    with pytest.raises(_native.TsbError) as e:
        _native.plan_compile_host(0, rects, n)
    assert e.value.code != _native.TSB_OK
    # dequantising pulls write f32/bf16/f16 only
    q = torch.zeros(8, 16, dtype=E4M3)
    s = torch.ones(8, 1)
    rects, n = build_rects([(StridedMem.from_tensor(q), StridedMem.from_tensor(torch.zeros(8, 16)))])
    rects[0].dst_dtype = _native.TSB_I8
    dq = _native.make_dq_source_array(1)
    dq[0] = _native.DqSource(q.data_ptr(), s.data_ptr(), 1, 8, 16, 0, 0, _native.TSB_SCALE_PER_CHANNEL, 0)
    expect(_native.TSB_ERR_INVALID, lambda: _native.dequant_fp8_compile_host(0, rects, n, dq, 1), "dequantising")
    # requantising pulls read and write float8_e4m3fn
    rects[0].src_dtype, rects[0].dst_dtype = _native.TSB_F8E4M3, _native.TSB_I8
    tg = _native.make_sq_target_array(1)
    tg[0] = _native.SqTarget(dst.data_ptr(), s.data_ptr(), 1, 8, 16, _native.TSB_SCALE_PER_CHANNEL, 0)
    expect(_native.TSB_ERR_INVALID, lambda: _native.requant_fp8_compile_host(0, rects, n, dq, 1, tg, 1), "float8_e4m3fn")
    # source-side quantisation reads f32/bf16/f16 only
    st = _native.make_source_quant_target_array(1)
    st[0] = _native.SourceQuantTarget(dst.data_ptr(), q.data_ptr(), s.data_ptr(), 1, 8, 16, 0, 0, _native.TSB_I8,
                                      _native.TSB_SCALE_PER_CHANNEL)
    with pytest.raises(_native.TsbError):
        _native.source_quant_compile_host(0, st, 1)


# ---- Python routing and refusals, before any device work ---------------------------------------------------------
no_export = pytest.fixture(no_export)


def scale_for(g):
    return torch.zeros({"block": (2, 2), "channel": (256, 1), "tensor": ()}[g])


@pytest.mark.parametrize("g", GRANULARITIES)
def test_int8_destinations_take_the_quantise_route(g):
    for dtype in (torch.bfloat16, torch.float16, torch.float32):
        d = fake_dest(torch.int8)
        out = DirectWeightSyncDest._check_scales({"w": [scaled_handle(dtype)] * 2}, {"w": d}, {KW[g]: {"w": scale_for(g)}})
        assert out["w"][0] == KW[g] and out["w"][1] is d and out["w"][3] == "quantise"


@pytest.mark.parametrize("g", GRANULARITIES)
def test_scaled_fp8_handles_into_int8_are_refused(g):
    for kw in ({}, {"requantize": True}, {"verbatim": True}):
        with pytest.raises(TypeError, match="int8 destinations are quantised from bf16, f16 or f32 handles"):
            DirectWeightSyncDest._check_scales({"w": [scaled_handle(E4M3, g)]}, {"w": fake_dest(torch.int8)},
                                               {KW[g]: {"w": scale_for(g)}}, **kw)


def test_int8_handles_need_one_float_dtype():
    for handles in ([scaled_handle(torch.int8)], [scaled_handle(E4M3)],
                    [scaled_handle(torch.bfloat16), scaled_handle(torch.float32)]):
        with pytest.raises(TypeError, match="read bf16, f16 or f32 handles of one dtype"):
            DirectWeightSyncDest._check_scales({"w": handles}, {"w": fake_dest(torch.int8)},
                                               {"channel_scales": {"w": scale_for("channel")}}, requantize=True)


def test_other_destination_dtypes_are_still_refused():
    for dtype in (torch.uint8, torch.float8_e5m2, torch.bfloat16, torch.int16):
        with pytest.raises(TypeError, match="must be float8_e4m3fn or int8"):
            DirectWeightSyncDest._check_scales({"w": [scaled_handle(torch.bfloat16)]}, {"w": fake_dest(dtype)},
                                               {"block_scales": {"w": scale_for("block")}})


def test_scale_fmt_with_an_int8_destination_is_refused(no_export, monkeypatch):
    d = DirectWeightSyncDest()
    monkeypatch.setattr(DirectWeightSyncDest, "_build_plan", lambda *a, **k: (_ for _ in ()).throw(Boom("planned")))
    dest = fake_dest(torch.int8)
    with pytest.raises(ValueError, match="does not apply to int8 destinations"):
        asyncio.run(d.pull({"w": [scaled_handle(torch.bfloat16)]}, {"w": dest}, channel_scales={"w": scale_for("channel")},
                           scale_fmt="ue8m0"))
    assert d._plan is None


def test_store_path_still_refuses_the_scale_dicts():
    from torchstore_b200 import state_dict_utils

    for kw in ("block_scales", "channel_scales", "tensor_scales"):
        with pytest.raises(NotImplementedError, match="direct_rdma=True"):
            asyncio.run(state_dict_utils.get_state_dict(None, "k", {"w": torch.zeros(4, 4, dtype=torch.int8)},
                                                        **{kw: {"w": torch.zeros(1)}}))


def compile_spy(monkeypatch):
    """Monkeypatched builders: record (builder, device, targets' dst pointers, flags) instead of compiling."""
    from torchstore_b200 import direct_weight_sync as dws

    seen = []
    monkeypatch.setattr(dws.Plans, "build", classmethod(lambda cls, per_device: dws.Plans()))
    for name in ("build_block_fp8", "build_scaled_fp8", "build_requant_fp8"):
        monkeypatch.setattr(dws.Plans, name, classmethod(
            lambda cls, per_device, flags=0, name=name: seen.append(
                (name, {dev: [t.dst for t in args[-1]] for dev, args in per_device.items()}, flags)) or {0: len(seen)}))
    return seen


def test_mixed_pull_builds_separate_int8_plans(monkeypatch):
    seen = compile_spy(monkeypatch)
    d = DirectWeightSyncDest()
    d._plan = []

    def dest(dtype, ptr):
        return types.SimpleNamespace(dtype=dtype, device=torch.device("cuda", 0), shape=(256, 256), numel=lambda: 256 * 256,
                                     data_ptr=lambda: ptr)

    scaled = {"fb": ("block_scales", dest(E4M3, 1), torch.zeros(2, 2)),
              "ib": ("block_scales", dest(torch.int8, 2), torch.zeros(2, 2)),
              "fc": ("channel_scales", dest(E4M3, 3), torch.zeros(256, 1)),
              "it": ("tensor_scales", dest(torch.int8, 4), torch.zeros(())),
              "ic": ("channel_scales", dest(torch.int8, 5), torch.zeros(256, 1))}
    d._compile(scaled, set(), set(), 0)
    assert seen == [("build_block_fp8", {0: [1]}, 0), ("build_scaled_fp8", {0: [3]}, 0),
                    ("build_block_fp8", {0: [2]}, 0), ("build_scaled_fp8", {0: [4, 5]}, 0)]
    assert d._block_plans and d._scaled_plans and d._int8_block_plans and d._int8_scaled_plans
    assert d._int8_block_plans in d._fp8_plans and d._int8_scaled_plans in d._fp8_plans
    assert {id(p) for p in d._fp8_plans} >= {id(d._int8_block_plans), id(d._int8_scaled_plans)}


@pytest.mark.parametrize("built,now", [(E4M3, torch.int8), (torch.int8, E4M3)])
def test_plan_rebuilds_on_a_dtype_flip(monkeypatch, built, now):
    """A cached plan is dropped when a scaled name's destination changes between float8_e4m3fn and int8, even at
    the same address (the caching allocator hands a freed block straight back), and kept while it does not.  The
    plans are built by pull() itself, with planning and the native builders stubbed out."""
    from torchstore_b200 import direct_weight_sync as dws

    plans_built = []
    monkeypatch.setattr(DirectWeightSyncDest, "_build_plan", lambda self, *a, **k: plans_built.append(1) or [])
    monkeypatch.setattr(dws.Plans, "build", classmethod(lambda cls, per_device: dws.Plans()))
    monkeypatch.setattr(dws.Plans, "build_scaled_fp8", classmethod(lambda cls, per_device, flags=0: dws.Plans()))
    handles = {"w": [scaled_handle(torch.bfloat16)]}
    scales = {"w": scale_for("channel")}
    d = DirectWeightSyncDest()
    asyncio.run(d.pull(handles, {"w": fake_dest(built)}, channel_scales=scales))
    asyncio.run(d.pull(handles, {"w": fake_dest(built)}, channel_scales=scales))  # another wrapper, same memory
    assert len(plans_built) == 1
    asyncio.run(d.pull(handles, {"w": fake_dest(now)}, channel_scales=scales))  # same address, other dtype
    assert len(plans_built) == 2
    asyncio.run(d.pull(handles, {"w": fake_dest(now)}, channel_scales=scales))
    assert len(plans_built) == 2
    d.close()

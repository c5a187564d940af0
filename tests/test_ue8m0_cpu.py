"""Power-of-two (UE8M0) scales without a GPU: the scale step's edge cases in numpy and torch, the numpy oracle
pinned to torch CPU's fixture, the C-ABI's TSB_QUANT_UE8M0 flag (accepted by the four quantising kinds with
identical tables, refused elsewhere), their compiled tables replayed on host memory against the formula, and the
Python validation of ``scale_fmt``."""

import asyncio
import os
import types

import numpy as np
import pytest
import torch

from oracle.ue8m0_oracle import (GRANULARITIES, bits_of, digest, edge_amaxes, fixture_inputs, log2_scale_inv, quantize,
                                 replay_block, replay_requant, replay_scaled, replay_source, requantize, scales_of_amax,
                                 synth_f32, torch_quantize, torch_scales_of_amax, widen)
from tests.helpers import Boom, expect_invalid, no_export
from torchstore_b200 import _native
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource
from torchstore_b200.planner import StridedMem, build_rects

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "ue8m0_vectors.npz")
E4M3 = torch.float8_e4m3fn
CODE = {"block": _native.TSB_SCALE_PER_BLOCK, "channel": _native.TSB_SCALE_PER_CHANNEL, "tensor": _native.TSB_SCALE_PER_TENSOR}
DT = {torch.bfloat16: _native.TSB_BF16, torch.float16: _native.TSB_F16, torch.float32: _native.TSB_F32}
UE8M0 = _native.TSB_QUANT_UE8M0
F32 = np.float32


def u32(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def is_pow2(a: np.ndarray) -> np.ndarray:
    return (u32(a) & 0x007FFFFF) == 0


# ---- the scale step --------------------------------------------------------------------------------------------
def test_step_edge_cases():
    cases = [  # amax -> scale_inv
        (F32(0), F32(2.0 ** -22)),  # clamped to 1e-4: t = 2.23e-7, up to 2^-22
        (F32(1e-5), F32(2.0 ** -22)),
        (F32(448 * 2.0 ** -3), F32(2.0 ** -3)),  # 448 * 2^k exactly: 2^k
        (F32(448), F32(1)),
        (F32(448 * 2.0 ** 20), F32(2.0 ** 20)),
        (np.nextafter(F32(448), F32(np.inf)), F32(2)),  # 448 * 2^k * (1 + 2^-23): 2^(k+1)
        (np.nextafter(F32(448 * 2.0 ** 7), F32(np.inf)), F32(2.0 ** 8)),
        (np.nextafter(F32(896), F32(0)), F32(2)),  # just below 448 * 2^(k+1): 2^(k+1)
        (np.nextafter(F32(448 * 2.0 ** -9), F32(0)), F32(2.0 ** -9)),
        (np.finfo(np.float32).max, F32(2.0 ** 120)),
        (F32(np.inf), F32(np.inf)),
    ]
    amax = np.array([a for a, _ in cases], dtype=np.float32)
    want = np.array([w for _, w in cases], dtype=np.float32)
    scale, scale_inv = scales_of_amax(amax)
    assert np.array_equal(u32(scale_inv), u32(want))
    assert np.array_equal(u32(scale), u32(np.float32(1) / want))  # exact: 0 for Inf
    assert scale[-1] == 0
    tscale, tscale_inv = torch_scales_of_amax(torch.from_numpy(amax))
    assert np.array_equal(u32(tscale_inv.numpy()), u32(scale_inv)) and np.array_equal(u32(tscale.numpy()), u32(scale))
    nan_scale, nan_inv = scales_of_amax(np.array([np.nan], dtype=np.float32))
    assert np.isnan(nan_scale).all() and np.isnan(nan_inv).all()
    assert torch.isnan(torch.cat(torch_scales_of_amax(torch.tensor([float("nan")])))).all()


def test_step_is_the_smallest_power_of_two_not_below_t():
    a = np.concatenate([edge_amaxes(), np.abs(synth_f32((4096,), 5, spread=60).numpy())]).astype(np.float32)
    t = (np.maximum(a, F32(1e-4)) / F32(448)).astype(np.float32)
    scale, scale_inv = scales_of_amax(a)
    assert is_pow2(scale_inv).all() and is_pow2(scale).all()
    assert (t <= scale_inv).all() and (scale_inv < 2 * t.astype(np.float64)).all()
    assert np.array_equal(u32(torch_scales_of_amax(torch.from_numpy(a))[1].numpy()), u32(scale_inv))
    # |x * scale| <= 448 for |x| <= amax: the narrowing never saturates
    assert (a.astype(np.float64) * scale <= 448).all()


def test_log2_rendering_differs_near_powers_of_two():
    """2 ** ceil(log2(t)) picks one power too small where t sits within float32 rounding above a power of two:
    the reason the rule is pinned on t's bits."""
    t = (np.maximum(edge_amaxes(), F32(1e-4)) / F32(448)).astype(np.float32)
    bitwise = scales_of_amax(edge_amaxes())[1]
    log2 = log2_scale_inv(t)
    differ = u32(log2) != u32(bitwise)
    assert differ.any()
    assert (log2[differ] < t[differ]).all()  # too small: its quantised bytes can exceed 448 before the narrowing


def test_quantised_bytes_stay_within_448():
    x = synth_f32((300, 260), 3, spread=30)
    for g in GRANULARITIES:
        for r0, c0 in ((0, 0), (37, 70)):
            q, s = quantize(x.numpy(), g, r0, c0, scale_fmt="ue8m0")
            y = torch.from_numpy(q).view(E4M3).float().abs()
            assert y.max() <= 448 and is_pow2(s).all()
            # None is the float32 formula, unchanged
            q0, s0 = quantize(x.numpy(), g, r0, c0)
            from oracle.source_quant_oracle import quantize as f32_quantize

            w0, ws0 = f32_quantize(x.numpy(), g, r0, c0)
            assert np.array_equal(q0, w0) and np.array_equal(u32(s0), u32(ws0))


@pytest.mark.parametrize("g", GRANULARITIES)
def test_torch_rendering_matches_the_oracle(g):
    for dtype in (torch.bfloat16, torch.float16, torch.float32):
        x = synth_f32((3, 130, 260), 17).to(dtype)
        for r0, c0 in ((0, 0), (100, 5)):
            q, s = quantize(widen(bits_of(x), str(dtype)[6:]), g, r0, c0, scale_fmt="ue8m0")
            tq, ts = torch_quantize(x, g, r0, c0, scale_fmt="ue8m0")
            assert np.array_equal(tq.view(torch.uint8).numpy(), q) and np.array_equal(u32(ts.numpy()), u32(s))


def test_unknown_scale_fmt_is_refused_by_the_oracle():
    with pytest.raises(ValueError, match="scale_fmt"):
        quantize(np.zeros((2, 2), np.float32), "block", scale_fmt="e8m0")


# ---- the fixture -------------------------------------------------------------------------------------------------
def fixture_cases():
    d = np.load(GOLDEN)
    inputs = {name: (x, g, r0, c0) for name, x, g, r0, c0 in fixture_inputs()}
    out = []
    for i, name in enumerate(d["names"]):
        x, g, r0, c0 = inputs[str(name)]
        want_q = d[f"q{i}"] if f"q{i}" in d.files else str(d[f"q_sha{i}"])
        out.append((str(name), widen(bits_of(x), str(d[f"dtype{i}"])), g, r0, c0, want_q, d[f"s{i}"]))
    return out


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
    """Bit-exact; NaN scales and the bytes of non-finite groups NaN-agnostically (their NaN encoding is the
    platform's)."""
    name, x, g, r0, c0, want_q, want_s = case
    q, s = quantize(x, g, r0, c0, scale_fmt="ue8m0")
    assert s.shape == want_s.shape
    assert np.array_equal(np.isnan(s), np.isnan(want_s))
    fin = ~np.isnan(want_s)
    assert np.array_equal(u32(s)[fin], u32(want_s)[fin])
    assert is_pow2(s[np.isfinite(s)]).all()
    if isinstance(want_q, str):
        assert digest(q) == want_q
    else:
        nan_q, nan_w = (q & 0x7F) == 0x7F, (want_q & 0x7F) == 0x7F
        assert np.array_equal(nan_q, nan_w) and np.array_equal(q[~nan_w], want_q[~nan_w])
    if name.endswith("nonfinite") and g != "tensor":
        assert np.isinf(s).any() and np.isnan(s).any()


def test_fixture_reaches_the_edges():
    cases = {c[0]: c for c in fixture_cases()}
    _, _, _, _, _, _, s = cases["channel_float32_edges"]
    want = scales_of_amax(edge_amaxes())[1]
    assert np.array_equal(u32(s.reshape(-1)), u32(want))
    for g in GRANULARITIES:
        for dtype in ("bfloat16", "float16", "float32"):
            assert {f"{g}_{dtype}_300x200_at_0_0", f"{g}_{dtype}_300x200_at_37_70", f"{g}_{dtype}_moe_3x130x260"} <= set(cases)


# ---- the C-ABI ---------------------------------------------------------------------------------------------------
def test_abi_version_is_9():
    assert _native.TSB_ABI_VERSION == 9 and _native.lib().tsb_abi_version() == 9


def host_pull(full: torch.Tensor, cuts, dest_dtype=E4M3):
    """Row shards ``full[a:b]`` of a host tensor pulled into one whole-tensor destination: (dest, rects, n, keep)."""
    dest = torch.full(full.shape, 0x55, dtype=torch.uint8).view(dest_dtype)
    shards = [full[a:b].contiguous() for a, b in cuts]
    d = StridedMem.from_tensor(dest)
    pairs = [(StridedMem.from_tensor(s), d.sub((slice(a, b), slice(None)))) for s, (a, b) in zip(shards, cuts)]
    rects, n = build_rects(pairs)
    return dest, rects, n, shards


def block_case(flags):
    full = synth_f32((300, 260), 11).to(torch.bfloat16)
    dest, rects, n, keep = host_pull(full, ((0, 150), (150, 300)))
    scale = torch.full((3, 3), -1.0)
    tg = _native.make_target_array(1)
    tg[0] = _native.BqTarget(dest.data_ptr(), scale.data_ptr(), 1, 300, 260)
    compile_ = lambda f: _native.block_fp8_compile_host(0, rects, n, tg, 1, f)  # noqa: E731
    return full, "block", dest, scale, compile_(flags), (keep, rects, tg, compile_)


def scaled_case(g, cols, flags):
    full = synth_f32((40, cols), 12).to(torch.bfloat16)
    dest, rects, n, keep = host_pull(full, ((0, 13), (13, 40)))
    scale = torch.full((40, 1) if g == "channel" else (), -1.0)
    tg = _native.make_sq_target_array(1)
    tg[0] = _native.SqTarget(dest.data_ptr(), scale.data_ptr(), 1, 40, cols, CODE[g], 0)
    compile_ = lambda f: _native.scaled_fp8_compile_host(0, rects, n, tg, 1, f)  # noqa: E731
    return full, g, dest, scale, compile_(flags), (keep, rects, tg, compile_)


def source_case(g, flags):
    x = synth_f32((300, 200), 13).to(torch.float16)
    bits = bits_of(x)
    q = np.full(x.shape, 0xAB, dtype=np.uint8)
    from torchstore_b200.direct_weight_sync import source_scale_shapes

    s = np.full(source_scale_shapes(g, tuple(x.shape), 37, 70)[0], np.nan, dtype=np.float32)
    tg = _native.make_source_quant_target_array(1)
    tg[0] = _native.SourceQuantTarget(bits.ctypes.data, q.ctypes.data, s.ctypes.data, 1, 300, 200, 37, 70, _native.TSB_F16, CODE[g])
    compile_ = lambda f: _native.source_quant_compile_host(0, tg, 1, f)  # noqa: E731
    return x, q, s, compile_(flags), (bits, tg, compile_)


def requant_case(dg, flags):
    """Two block-scaled fp8 row shards (rows 0..100 and 100..192: block row 0 straddles them) into a whole
    ``dg``-scaled destination."""
    gen = torch.Generator().manual_seed(3)
    q_full = (torch.randn(192, 160, generator=gen) * 40).to(E4M3)
    s_full = torch.rand(2, 2, generator=gen) * 0.01 + 1e-3
    cuts = ((0, 100), (100, 192))
    dest, rects, n, shards = host_pull(q_full, cuts)
    for i in range(n):
        rects[i].src_dtype = rects[i].dst_dtype = _native.TSB_F8E4M3
    scales = [s_full[a // 128: -(-b // 128)].contiguous() for a, b in cuts]
    src = _native.make_dq_source_array(2)
    for i, ((a, b), sh, sc) in enumerate(zip(cuts, shards, scales)):
        src[i] = _native.DqSource(sh.data_ptr(), sc.data_ptr(), 1, b - a, 160, a, 0, _native.TSB_SCALE_PER_BLOCK, 0)
    scale = torch.full({"block": (2, 2), "channel": (192, 1), "tensor": ()}[dg], -1.0)
    tg = _native.make_sq_target_array(1)
    tg[0] = _native.SqTarget(dest.data_ptr(), scale.data_ptr(), 1, 192, 160, CODE[dg], 0)
    compile_ = lambda f: _native.requant_fp8_compile_host(0, rects, n, src, 2, tg, 1, f)  # noqa: E731
    return q_full, s_full, dest, scale, compile_(flags), (shards, scales, rects, src, tg, compile_)


def same_tables(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        if isinstance(x, np.ndarray):
            assert x.dtype == y.dtype and x.tobytes() == y.tobytes()
        else:
            assert x == y


def test_quantising_kinds_accept_the_flag_with_identical_tables():
    cases = [block_case(0)] + [scaled_case(g, c, 0) for g, c in (("channel", 260), ("channel", 16400), ("tensor", 260))]
    cases += [source_case(g, 0) for g in GRANULARITIES] + [requant_case(g, 0) for g in GRANULARITIES]
    for case in cases:
        compile_ = case[-1][-1]
        same_tables(compile_(0), compile_(UE8M0))


def test_unknown_bits_and_the_dequantising_kind_are_refused():
    for bad in (2, 1 << 31, UE8M0 | 4):
        expect_invalid(lambda: block_case(bad), "flags must be")
        expect_invalid(lambda: scaled_case("channel", 260, bad), "flags must be")
        expect_invalid(lambda: source_case("block", bad), "flags must be")
        expect_invalid(lambda: requant_case("block", bad), "flags must be")
    q = torch.zeros(8, 16, dtype=E4M3)
    s = torch.ones(8, 1)
    y = torch.zeros(8, 16)
    rects, n = build_rects([(StridedMem.from_tensor(q), StridedMem.from_tensor(y))])
    src = _native.make_dq_source_array(1)
    src[0] = _native.DqSource(q.data_ptr(), s.data_ptr(), 1, 8, 16, 0, 0, _native.TSB_SCALE_PER_CHANNEL, 0)
    assert len(_native.dequant_fp8_compile_host(0, rects, n, src, 1)) == 1
    for bad in (UE8M0, 2):
        expect_invalid(lambda: _native.dequant_fp8_compile_host(0, rects, n, src, 1, bad), "flags must be")
        # plan creation checks the flags before it touches a device
        expect_invalid(lambda: _native.dequant_fp8_plan_create(0, rects, n, [src[0]], flags=bad), "flags must be")
    expect_invalid(lambda: _native.block_fp8_plan_create(0, rects, n, [], flags=2), "flags must be")


def test_replayed_block_and_scaled_tables_match_the_formula():
    for fmt, flags in ((None, 0), ("ue8m0", UE8M0)):
        cases = [block_case(flags)] + [scaled_case(g, c, flags) for g, c in (("channel", 260), ("channel", 16400), ("tensor", 260))]
        for full, g, dest, scale, tables, _keep in cases:
            (replay_block if g == "block" else replay_scaled)(*tables, scale_fmt=fmt)
            want_q, want_s = quantize(full.float().numpy(), g, scale_fmt=fmt)
            assert np.array_equal(dest.view(torch.uint8).numpy(), want_q), (g, fmt)
            assert np.array_equal(u32(scale.numpy()), u32(want_s)), (g, fmt)
            if fmt:
                assert is_pow2(scale.numpy()).all()


@pytest.mark.parametrize("g", GRANULARITIES)
def test_replayed_source_tables_match_the_formula(g):
    x, q, s, tables, _keep = source_case(g, UE8M0)
    replay_source(*tables, scale_fmt="ue8m0")
    want_q, want_s = quantize(widen(bits_of(x), "float16"), g, 37, 70, scale_fmt="ue8m0")
    assert np.array_equal(q, want_q) and np.array_equal(u32(s), u32(want_s))


@pytest.mark.parametrize("dg", GRANULARITIES)
def test_replayed_requant_tables_match_the_formula(dg):
    q_full, s_full, dest, scale, tables, _keep = requant_case(dg, UE8M0)
    replay_requant(*tables, scale_fmt="ue8m0")
    want_q, want_s = requantize(q_full.view(torch.uint8).numpy(), s_full.numpy(), "block", 0, 0, dg, scale_fmt="ue8m0")
    assert np.array_equal(dest.view(torch.uint8).numpy(), want_q)
    assert np.array_equal(u32(scale.numpy()).reshape(-1), u32(want_s).reshape(-1))


def test_requantising_power_of_two_groups_onto_themselves_is_lossless():
    """UE8M0 block source groups requantised into coinciding UE8M0 destination groups keep every value."""
    x = synth_f32((256, 384), 21, spread=12).numpy()
    q, s = quantize(x, "block", scale_fmt="ue8m0")
    q2, s2 = requantize(q, s, "block", 0, 0, "block", scale_fmt="ue8m0")
    from oracle.dequant_fp8_oracle import dequantize

    before = dequantize(q, s, "block", dst="float32").view(np.float32)
    after = dequantize(q2, s2, "block", dst="float32").view(np.float32)
    assert np.array_equal(before, after) and (s2 <= s).all()


# ---- Python validation, before any device work -------------------------------------------------------------------
no_export = pytest.fixture(no_export)


@pytest.mark.parametrize("fmt", ["e8m0", "UE8M0", "", 1, "float32"])
def test_unknown_scale_fmt_is_refused(no_export, fmt):
    dest = DirectWeightSyncDest()
    with pytest.raises(ValueError, match="scale_fmt must be None or 'ue8m0'"):
        asyncio.run(dest.pull({}, {}, block_scales={"w": torch.zeros(1, 1)}, scale_fmt=fmt))
    src = DirectWeightSyncSource()
    with pytest.raises(ValueError, match="scale_fmt must be None or 'ue8m0'"):
        src.register({"w": torch.zeros(4, 4)}, rank=0, quantize={"w": "block"}, scale_fmt=fmt)
    assert dest._plan is None and src._handles == {} and not src._quant_plans


def test_scale_fmt_without_scaled_names_is_refused(no_export):
    with pytest.raises(ValueError, match="must name at least one"):
        asyncio.run(DirectWeightSyncDest().pull({}, {"w": torch.zeros(4, 4)}, scale_fmt="ue8m0"))
    with pytest.raises(ValueError, match="must name at least one"):
        asyncio.run(DirectWeightSyncDest().pull({}, {}, block_scales={}, scale_fmt="ue8m0"))
    src = DirectWeightSyncSource()
    with pytest.raises(ValueError, match="needs quantize"):
        src.register({"w": torch.zeros(4, 4)}, rank=0, scale_fmt="ue8m0")
    with pytest.raises(ValueError, match="needs quantize"):
        src.register({"w": torch.zeros(4, 4)}, rank=0, quantize={}, scale_fmt="ue8m0")
    assert src._handles == {}


def test_scale_fmt_is_validated_before_the_quantize_dict(no_export):
    with pytest.raises(ValueError, match="scale_fmt must be"):
        DirectWeightSyncSource().register({"w": torch.zeros(4, 4)}, rank=0, quantize={"nope": "block"}, scale_fmt="x")


def test_plan_cache_key_includes_the_scale_format():
    """A cached plan is rebuilt whenever scale_fmt changes, in either direction."""
    for built, fmt in ((None, "ue8m0"), ("ue8m0", None)):
        d = DirectWeightSyncDest()
        d._plan = []
        d._plan_key = (frozenset({("w", "block_scales")}), False, built)
        d.close = lambda: (_ for _ in ()).throw(Boom("rebuilt"))
        with pytest.raises(Boom):
            asyncio.run(d.pull({}, {}, block_scales={"w": torch.zeros(1, 1)}, scale_fmt=fmt))


def test_scale_fmt_reaches_the_plan_builders(monkeypatch):
    """pull() hands TSB_QUANT_UE8M0 to the quantising and requantising builders, and 0 without scale_fmt."""
    from torchstore_b200 import direct_weight_sync as dws

    seen = []
    d = DirectWeightSyncDest()
    d._plan = []
    monkeypatch.setattr(dws.Plans, "build", classmethod(lambda cls, per_device: dws.Plans()))
    monkeypatch.setattr(dws.Plans, "build_block_fp8", classmethod(lambda cls, per_device, flags=0: seen.append(flags) or {}))
    monkeypatch.setattr(dws.Plans, "build_requant_fp8", classmethod(lambda cls, per_device, flags=0: seen.append(flags) or {}))
    dest = types.SimpleNamespace(device=torch.device("cpu"), shape=(4, 4), numel=lambda: 16, data_ptr=lambda: 0)
    for flags in (UE8M0, 0):
        d._compile({"w": ("block_scales", dest, torch.zeros(1, 1)), "v": ("block_scales", dest, torch.zeros(1, 1))}, set(),
                   {"v"}, flags)
        assert seen == [flags, flags]
        seen.clear()


def test_store_path_refuses_scale_fmt():
    from torchstore_b200 import state_dict_utils

    with pytest.raises(NotImplementedError, match="scale_fmt needs direct_rdma=True"):
        asyncio.run(state_dict_utils.get_state_dict(None, "k", {"w": torch.zeros(1)}, scale_fmt="ue8m0"))
    with pytest.raises(NotImplementedError, match="scale_fmt needs direct_rdma=True"):
        asyncio.run(state_dict_utils.put_state_dict(None, {"w": torch.zeros(1)}, "k", scale_fmt="ue8m0"))


def test_public_signatures_default_to_the_float32_formula():
    import inspect

    from torchstore_b200 import api, state_dict_utils

    for fn in (DirectWeightSyncSource.register, DirectWeightSyncDest.pull, api.put_state_dict, api.get_state_dict,
               state_dict_utils.put_state_dict, state_dict_utils.get_state_dict):
        assert inspect.signature(fn).parameters["scale_fmt"].default is None, fn

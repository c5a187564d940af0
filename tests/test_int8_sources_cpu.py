"""Scaled INT8 sources without a GPU: the numpy oracle pinned to torch CPU's fixture, the C-ABI additions
(TSB_I8 dequantising rects, tsb_source_quant_*_as) and their refusals, the compiled tables replayed on host memory
against the oracle, every cell of the pull route table for scaled int8 handles, register / put_state_dict
validation with nothing exported, and the plan rebuild when a destination flips between float8_e4m3fn and int8."""

import asyncio
import os
import types

import numpy as np
import pytest
import torch

from oracle.int8_source_oracle import (DSTS, GRANULARITIES, bits_of, dequant_inputs, dequantize, digest, int8_of,
                                       quant_inputs, quantize, replay_dequant, replay_source, scale_of, scale_shape,
                                       synth_f32, torch_dequantize, torch_quantize, widen)
from tests.helpers import Boom, fake_dest, no_export, scaled_handle
from torchstore_b200 import _native
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource
from torchstore_b200.planner import StridedMem, build_rects

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "int8_source_vectors.npz")
E4M3 = torch.float8_e4m3fn
CODE = {"block": _native.TSB_SCALE_PER_BLOCK, "channel": _native.TSB_SCALE_PER_CHANNEL,
        "tensor": _native.TSB_SCALE_PER_TENSOR}
KW = {"block": "block_scales", "channel": "channel_scales", "tensor": "tensor_scales"}
FLOATS = (torch.bfloat16, torch.float16, torch.float32)


def u32(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def same_scales(a, b) -> bool:
    """float32 scales equal as bits, NaN matching any NaN."""
    a, b = np.asarray(a, dtype=np.float32).reshape(-1), np.asarray(b, dtype=np.float32).reshape(-1)
    nan = np.isnan(a)
    return a.shape == b.shape and np.array_equal(nan, np.isnan(b)) and np.array_equal(u32(a)[~nan], u32(b)[~nan])


def expect(code, fn, needle):
    with pytest.raises(_native.TsbError, match=needle) as e:
        fn()
    assert e.value.code == code


# ---- the oracle against torch CPU's fixture ------------------------------------------------------------------------
def test_fixture_inputs_are_the_recorded_ones():
    d = np.load(GOLDEN)
    cases = quant_inputs()
    assert [c[0] for c in cases] == [str(n) for n in d["names"]]
    for i, (name, x, g, r0, c0) in enumerate(cases):
        assert str(d[f"granularity{i}"]) == g and d[f"offset{i}"].tolist() == [r0, c0], name
        assert digest(bits_of(x)) == str(d[f"x_sha{i}"]), name
    dq = dequant_inputs()
    assert [c[0] for c in dq] == [str(n) for n in d["dq_names"]]
    for i, (name, g, r0, c0, q, s) in enumerate(dq):
        assert digest(q.view(torch.uint8).numpy()) == str(d[f"dq_q_sha{i}"]), name
        assert digest(s.numpy().view(np.uint32)) == str(d[f"dq_s_sha{i}"]), name


@pytest.mark.parametrize("i", range(45))
def test_quantising_oracle_matches_the_torch_cpu_fixture(i):
    d = np.load(GOLDEN)
    name, x, g, r0, c0 = quant_inputs()[i]
    q, s = quantize(widen(bits_of(x), str(x.dtype)[6:]), g, r0, c0)
    assert digest(q.view(np.uint8)) == str(d[f"q_sha{i}"]), name
    assert same_scales(s, d[f"s{i}"]), name
    assert q.min() >= -127  # symmetric: a finite group never reaches -128


@pytest.mark.parametrize("i", range(10))
def test_dequantising_oracle_matches_the_torch_cpu_fixture(i):
    d = np.load(GOLDEN)
    name, g, r0, c0, q, s = dequant_inputs()[i]
    for dst in DSTS:
        assert digest(dequantize(q.numpy(), s.numpy(), g, r0, c0, dst)) == str(d[f"dq_{dst}_sha{i}"]), (name, dst)


def test_torch_rendering_matches_the_oracle_on_odd_shapes():
    for g in GRANULARITIES:
        for shape, r0, c0 in (((1, 1), 0, 0), ((129, 3), 127, 1), ((2, 5, 257), 300, 129)):
            x = synth_f32(shape, 5)
            q, s = quantize(x.numpy(), g, r0, c0)
            tq, ts = torch_quantize(x, g, r0, c0)
            assert np.array_equal(q, tq.numpy()) and same_scales(s, ts.numpy())
            qi = int8_of(shape, 6)
            sc = scale_of(scale_shape(g, shape, r0, c0), 7)
            for dst in DSTS:
                assert np.array_equal(dequantize(qi.numpy(), sc.numpy(), g, r0, c0, dst),
                                      bits_of(torch_dequantize(qi, sc, g, r0, c0, getattr(torch, dst))))


# ---- source-side quantisation: tsb_source_quant_*_as ---------------------------------------------------------------
def sq_case(g, shape, dtype, r0, c0, seed=3):
    """A host shard and its int8 staging -> (x, q, s, targets)."""
    x = synth_f32(shape, seed).to(dtype)
    q = torch.full(shape, 0x55, dtype=torch.uint8).view(torch.int8)
    s = torch.full(scale_shape(g, shape, r0, c0), -1.0)
    rows, cols = shape[-2:]
    t = _native.make_source_quant_target_array(1)
    t[0] = _native.SourceQuantTarget(x.data_ptr(), q.data_ptr(), s.data_ptr(), x.numel() // (rows * cols), rows, cols,
                                     r0, c0, _native.cast_code(dtype), CODE[g])
    return x, q, s, t


# (granularity, shape, offset): units, mid-block shard offsets, an MoE stack, per-channel rows long enough for the
# two-pass path, per-tensor (two-pass)
SQ_REGIMES = (("block", (300, 260), (0, 0)), ("block", (200, 300), (37, 70)), ("block", (3, 130, 260), (100, 5)),
              ("channel", (40, 260), (13, 0)), ("channel", (6, 16400), (0, 0)), ("channel", (2, 20, 100), (5, 3)),
              ("tensor", (40, 260), (0, 0)), ("tensor", (3, 50, 70), (64, 64)))


@pytest.mark.parametrize("dtype", FLOATS, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("g,shape,offset", SQ_REGIMES)
def test_source_quant_tables_replay_to_the_oracle(g, shape, offset, dtype):
    x, q, s, t = sq_case(g, shape, dtype, *offset)
    units, tiles, n_groups = _native.source_quant_compile_host(0, t, 1, dst_dtype=_native.TSB_I8)
    assert (len(tiles) > 0) == (g == "tensor" or shape[-1] == 16400)
    replay_source(units, tiles, n_groups)
    want_q, want_s = quantize(widen(bits_of(x), str(dtype)[6:]), g, *offset)
    assert np.array_equal(q.numpy(), want_q) and same_scales(s.numpy(), want_s)


@pytest.mark.parametrize("g,shape,offset", SQ_REGIMES)
def test_source_quant_tables_do_not_depend_on_the_staging_dtype(g, shape, offset):
    *_, t = sq_case(g, shape, torch.bfloat16, *offset)
    i8 = _native.source_quant_compile_host(0, t, 1, dst_dtype=_native.TSB_I8)
    for other in (_native.source_quant_compile_host(0, t, 1, dst_dtype=_native.TSB_F8E4M3),
                  _native.source_quant_compile_host(0, t, 1)):
        assert len(other) == len(i8) and other[-1] == i8[-1]
        assert all(a.tobytes() == b.tobytes() and a.dtype == b.dtype for a, b in zip(other[:-1], i8[:-1]))


def test_source_quant_as_refusals():
    *_, t = sq_case("channel", (8, 16), torch.bfloat16, 0, 0)
    for bad in (_native.TSB_U8, _native.TSB_F8E5M2, _native.TSB_BF16, 11):
        expect(_native.TSB_ERR_INVALID, lambda bad=bad: _native.source_quant_compile_host(0, t, 1, dst_dtype=bad),
               "dst_dtype must be TSB_F8E4M3 or TSB_I8")
    expect(_native.TSB_ERR_INVALID,
           lambda: _native.source_quant_compile_host(0, t, 1, _native.TSB_QUANT_UE8M0, dst_dtype=_native.TSB_I8),
           "TSB_QUANT_UE8M0")
    _native.source_quant_compile_host(0, t, 1, _native.TSB_QUANT_UE8M0, dst_dtype=_native.TSB_F8E4M3)
    for flags in (2, 4):  # the other flag bits stay refused
        expect(_native.TSB_ERR_INVALID, lambda f=flags: _native.source_quant_compile_host(0, t, 1, f, dst_dtype=_native.TSB_I8),
               "flags")
    # TSB_I8 stays refused as a source dtype
    t[0].src_dtype = _native.TSB_I8
    expect(_native.TSB_ERR_INVALID, lambda: _native.source_quant_compile_host(0, t, 1, dst_dtype=_native.TSB_I8), "src_dtype")


def test_new_calls_are_declared_bound_and_exported():
    header = open(os.path.join(os.path.dirname(os.path.dirname(__file__)), "include", "tstore_b200.h")).read()
    for name in ("tsb_source_quant_plan_create_as", "tsb_source_quant_compile_host_as"):
        assert name in _native.EXPORTED_SYMBOLS and f"int {name}(" in header
        assert getattr(_native.lib(), name) is not None
    assert _native.lib().tsb_abi_version() == 9


# ---- dequantising int8 sources: TSB_I8 rects of tsb_dequant_fp8_* --------------------------------------------------
def dq_case(g, shape, r0, c0, dst_dtype, cuts):
    """Row shards [a, b) of an int8 source at global (r0, c0) pulled into a destination -> (q, s, dest, rects, n,
    sources, keep)."""
    q = int8_of(shape, 11)
    s = scale_of(scale_shape(g, shape, r0, c0), 12)
    dest = torch.zeros(shape, dtype=dst_dtype)
    qm, dm = StridedMem.from_tensor(q), StridedMem.from_tensor(dest)
    lead = [slice(None)] * (len(shape) - 2)
    pairs = [(qm.sub(lead + [slice(a, b), slice(None)]), dm.sub(lead + [slice(a, b), slice(None)])) for a, b in cuts]
    rects, n = build_rects(pairs, dequantise=True)
    rows, cols = shape[-2:]
    src = _native.make_dq_source_array(1)
    src[0] = _native.DqSource(q.data_ptr(), s.data_ptr(), q.numel() // (rows * cols), rows, cols, r0, c0, CODE[g], 0)
    return q, s, dest, rects, n, src, (pairs,)


DQ_REGIMES = (("block", (300, 260), 37, 70), ("block", (3, 130, 260), 100, 5), ("channel", (40, 260), 13, 0),
              ("tensor", (2, 40, 260), 0, 0))


@pytest.mark.parametrize("dst", FLOATS, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("g,shape,r0,c0", DQ_REGIMES)
def test_dequant_tables_replay_to_the_oracle(g, shape, r0, c0, dst):
    q, s, dest, rects, n, src, _keep = dq_case(g, shape, r0, c0, dst, ((0, 17), (17, shape[-2])))
    assert n == 2 and all(rects[i].src_dtype == _native.TSB_I8 for i in range(n))
    replay_dequant(_native.dequant_fp8_compile_host(0, rects, n, src, 1))
    want = dequantize(q.numpy(), s.numpy(), g, r0, c0, str(dst)[6:])
    assert np.array_equal(bits_of(dest), want)


@pytest.mark.parametrize("g,shape,r0,c0", DQ_REGIMES)
def test_dequant_tables_are_the_fp8_tables(g, shape, r0, c0):
    *_, rects, n, src, _keep = dq_case(g, shape, r0, c0, torch.bfloat16, ((0, 17), (17, shape[-2])))
    i8 = _native.dequant_fp8_compile_host(0, rects, n, src, 1)
    for i in range(n):  # the same buffers, the rects relabelled float8_e4m3fn
        rects[i].src_dtype = _native.TSB_F8E4M3
    fp8 = _native.dequant_fp8_compile_host(0, rects, n, src, 1)
    assert fp8.dtype == i8.dtype and fp8.tobytes() == i8.tobytes()


def test_dequant_refusals():
    *_, rects, n, src, _keep = dq_case("channel", (40, 260), 0, 0, torch.float32, ((0, 17), (17, 40)))
    # one plan reads one source dtype
    rects[1].src_dtype = _native.TSB_F8E4M3
    expect(_native.TSB_ERR_INVALID, lambda: _native.dequant_fp8_compile_host(0, rects, n, src, 1), "one source dtype")
    rects[0].src_dtype, rects[1].src_dtype = _native.TSB_F8E4M3, _native.TSB_I8
    expect(_native.TSB_ERR_INVALID, lambda: _native.dequant_fp8_compile_host(0, rects, n, src, 1), "one source dtype")
    # TSB_I8 stays refused as a destination, and other source codes stay refused
    rects[0].src_dtype = rects[1].src_dtype = _native.TSB_I8
    rects[0].dst_dtype = _native.TSB_I8
    expect(_native.TSB_ERR_INVALID, lambda: _native.dequant_fp8_compile_host(0, rects, n, src, 1), "dequantising")
    rects[0].dst_dtype = _native.TSB_F32
    for bad in (_native.TSB_U8, _native.TSB_F8E5M2, _native.TSB_BF16):
        rects[0].src_dtype = rects[1].src_dtype = bad
        expect(_native.TSB_ERR_INVALID, lambda: _native.dequant_fp8_compile_host(0, rects, n, src, 1), "float8_e4m3fn or int8")
    rects[0].src_dtype = rects[1].src_dtype = _native.TSB_I8
    src[0].pad = 1
    expect(_native.TSB_ERR_INVALID, lambda: _native.dequant_fp8_compile_host(0, rects, n, src, 1), "pad")
    src[0].pad = 0
    _native.dequant_fp8_compile_host(0, rects, n, src, 1)
    expect(_native.TSB_ERR_INVALID,
           lambda: _native.dequant_fp8_compile_host(0, rects, n, src, 1, _native.TSB_QUANT_UE8M0), "flags")


def test_tsb_i8_stays_out_of_the_casts_the_copy_plan_and_requantising():
    lib = _native.lib()
    for other in (_native.TSB_F32, _native.TSB_BF16, _native.TSB_F16, _native.TSB_U8, _native.TSB_F8E4M3):
        assert lib.tsb_cast_supported(other, _native.TSB_I8) == 0 and lib.tsb_cast_supported(_native.TSB_I8, other) == 0
    q, dst = torch.zeros(8, 16, dtype=torch.int8), torch.zeros(8, 16)
    with pytest.raises(NotImplementedError, match="no fused cast kernel"):
        build_rects([(StridedMem.from_tensor(q), StridedMem.from_tensor(dst))])
    rects, n = build_rects([(StridedMem.from_tensor(q), StridedMem.from_tensor(dst))], dequantise=True)
    assert rects[0].src_dtype == _native.TSB_I8 and rects[0].dst_dtype == _native.TSB_F32
    with pytest.raises(_native.TsbError):
        _native.plan_compile_host(0, rects, n)
    rects, n = build_rects([(StridedMem.from_tensor(q), StridedMem.from_tensor(q.clone()))], dequantise=True)
    assert rects[0].src_dtype == rects[0].dst_dtype == _native.TSB_U8  # int8 -> int8 stays a byte move
    s = torch.ones(8, 1)
    dq = _native.make_dq_source_array(1)
    dq[0] = _native.DqSource(q.data_ptr(), s.data_ptr(), 1, 8, 16, 0, 0, _native.TSB_SCALE_PER_CHANNEL, 0)
    tg = _native.make_sq_target_array(1)
    tg[0] = _native.SqTarget(q.data_ptr(), s.data_ptr(), 1, 8, 16, _native.TSB_SCALE_PER_CHANNEL, 0)
    rects[0].src_dtype = rects[0].dst_dtype = _native.TSB_I8
    expect(_native.TSB_ERR_INVALID, lambda: _native.requant_fp8_compile_host(0, rects, n, dq, 1, tg, 1), "float8_e4m3fn")


# ---- the route table -----------------------------------------------------------------------------------------------
def scale_for(g):
    return torch.zeros({"block": (2, 2), "channel": (256, 1), "tensor": ()}[g])


def check_scales(handles, dest, g, **kw):
    return DirectWeightSyncDest._check_scales({"w": handles}, {"w": dest}, {KW[g]: {"w": scale_for(g)}}, **kw)


def check_dequant(handles, dest):
    return DirectWeightSyncDest._check_dequant({"w": handles}, {"w": dest}, {})


FLAGS = ({}, {"requantize": True}, {"verbatim": True})


@pytest.mark.parametrize("g", GRANULARITIES)
def test_int8_handles_into_floats_dequantise(g):
    for dtype in FLOATS:
        assert check_dequant([scaled_handle(torch.int8, g)] * 2, torch.zeros(4, 4, dtype=dtype)) == {"w"}


@pytest.mark.parametrize("g", GRANULARITIES)
def test_int8_handles_into_named_int8_move_verbatim_only(g):
    h = [scaled_handle(torch.int8, g)] * 2
    assert check_scales(h, fake_dest(torch.int8), g, verbatim=True)["w"][3] == "verbatim"
    with pytest.raises(TypeError, match="pass verbatim=True"):
        check_scales(h, fake_dest(torch.int8), g)
    with pytest.raises(TypeError, match="not requantised"):
        check_scales(h, fake_dest(torch.int8), g, requantize=True)
    other = "tensor" if g != "tensor" else "channel"
    with pytest.raises(ValueError, match="granularity only"):
        check_scales([scaled_handle(torch.int8, other)], fake_dest(torch.int8), g, verbatim=True)


@pytest.mark.parametrize("g", GRANULARITIES)
def test_int8_handles_into_unnamed_int8_are_bytes(g):
    assert check_dequant([scaled_handle(torch.int8, g)], torch.zeros(4, 4, dtype=torch.int8)) == set()


@pytest.mark.parametrize("g", GRANULARITIES)
def test_int8_handles_never_become_fp8(g):
    for kw in FLAGS:
        with pytest.raises(TypeError, match="int8 is not converted to fp8"):
            check_scales([scaled_handle(torch.int8, g)], fake_dest(E4M3), g, **kw)
    with pytest.raises(TypeError, match="int8 is not converted to fp8"):
        check_dequant([scaled_handle(torch.int8, g)], torch.zeros(4, 4, dtype=E4M3))


@pytest.mark.parametrize("dtype", (torch.uint8, torch.int16, torch.float64, torch.float8_e5m2), ids=str)
def test_int8_handles_into_other_dtypes_are_refused(dtype):
    with pytest.raises(TypeError, match="must be bfloat16, float16, float32"):
        check_dequant([scaled_handle(torch.int8, "channel")], torch.zeros(4, 4, dtype=dtype))
    with pytest.raises(TypeError, match="must be float8_e4m3fn or int8"):
        check_scales([scaled_handle(torch.int8, "channel")], fake_dest(dtype), "channel", verbatim=True)


def test_mixed_formats_and_mixed_scaling_are_refused():
    mixed = [scaled_handle(torch.int8, "channel"), scaled_handle(E4M3, "channel")]
    for kw in FLAGS:
        for dest in (fake_dest(torch.int8), fake_dest(E4M3)):
            with pytest.raises(ValueError, match="mix scaled int8 and scaled fp8"):
                check_scales(mixed, dest, "channel", **kw)
    with pytest.raises(ValueError, match="mix scaled int8 and scaled fp8"):
        check_dequant(mixed, torch.zeros(4, 4))
    half = [scaled_handle(torch.int8, "channel"), scaled_handle(torch.int8)]
    with pytest.raises(ValueError, match="mix scaled int8 and unscaled"):
        check_dequant(half, torch.zeros(4, 4))
    for kw in FLAGS:
        with pytest.raises(ValueError, match="mix scaled int8 and unscaled"):
            check_scales(half, fake_dest(torch.int8), "channel", **kw)


@pytest.mark.parametrize("g", GRANULARITIES)
def test_fp8_verdicts_are_unchanged(g):
    for kw in FLAGS:
        with pytest.raises(TypeError, match="int8 destinations are quantised from bf16, f16 or f32 handles"):
            check_scales([scaled_handle(E4M3, g)], fake_dest(torch.int8), g, **kw)
    assert check_scales([scaled_handle(E4M3, g)], fake_dest(E4M3), g, verbatim=True)["w"][3] == "verbatim"
    assert check_dequant([scaled_handle(E4M3, g)], torch.zeros(4, 4)) == {"w"}
    with pytest.raises(ValueError, match="mix scaled fp8 and unscaled"):
        check_dequant([scaled_handle(E4M3, g), scaled_handle(torch.bfloat16)], torch.zeros(4, 4))


# ---- refusals before anything is compiled ---------------------------------------------------------------------------
no_export = pytest.fixture(no_export)


def _w(*shape, dtype=torch.bfloat16):
    return torch.zeros(*shape, dtype=dtype)


@pytest.mark.parametrize("kw, exc, needle", [
    ({"quant_dtype": torch.int8}, ValueError, "needs quantize"),
    ({"quant_dtype": torch.int8, "quantize": {}}, ValueError, "needs quantize"),
    ({"quant_dtype": torch.float8_e5m2, "quantize": {"w": "block"}}, ValueError, "quant_dtype must be"),
    ({"quant_dtype": torch.bfloat16, "quantize": {"w": "block"}}, ValueError, "quant_dtype must be"),
    ({"quant_dtype": "int8", "quantize": {"w": "block"}}, ValueError, "quant_dtype must be"),
    ({"quant_dtype": torch.int8, "quantize": {"w": "block"}, "scale_fmt": "ue8m0"}, ValueError, "int8 staging"),
    ({"quant_dtype": torch.int8, "quantize": {"w": "row"}}, ValueError, "must be one of"),
    ({"quant_dtype": torch.int8, "quantize": {"w": "block"}}, ValueError, "must live on a CUDA device"),
    ({"block_scales": {"i": torch.zeros(1, 1)}}, ValueError, "CUDA tensor"),  # int8 passes the dtype check
    ({"block_scales": {"w": torch.zeros(1, 1)}}, TypeError, "must be float8_e4m3fn or int8, not torch.bfloat16"),
    ({"block_scales": {"i": torch.zeros(1, 1)}, "transfer_dtype": torch.float16}, ValueError, "transfer_dtype"),
])
def test_register_validation(no_export, kw, exc, needle):
    src = DirectWeightSyncSource()
    with pytest.raises(exc, match=needle):
        src.register({"w": _w(4, 4), "i": _w(4, 4, dtype=torch.int8)}, rank=0, **kw)
    assert src._handles == {} and src._quantized == {} and not src._quant_plans


def test_store_path_refuses_quant_dtype():
    from torchstore_b200 import state_dict_utils

    with pytest.raises(NotImplementedError, match="quant_dtype needs direct_rdma=True"):
        asyncio.run(state_dict_utils.put_state_dict(None, {"w": _w(4, 4)}, "k", quant_dtype=torch.int8))


def test_put_state_dict_passes_quant_dtype_through(monkeypatch):
    from torchstore_b200 import api, state_dict_utils

    seen = {}

    async def fake_put(**kw):
        seen.update(kw)

    async def fake_client(name):
        return None

    monkeypatch.setattr(state_dict_utils, "put_state_dict", fake_put)
    monkeypatch.setattr(api, "client", fake_client)
    asyncio.run(api.put_state_dict({"w": _w(4, 4)}, "k", direct_rdma=True, quantize={"w": "block"},
                                   quant_dtype=torch.int8))
    assert seen["quant_dtype"] is torch.int8 and seen["quantize"] == {"w": "block"}


def test_pull_refusals_come_before_planning(monkeypatch):
    d = DirectWeightSyncDest()
    monkeypatch.setattr(DirectWeightSyncDest, "_build_plan", lambda *a, **k: (_ for _ in ()).throw(Boom("planned")))
    h = {"w": [scaled_handle(torch.int8, "channel")]}
    with pytest.raises(TypeError, match="pass verbatim=True"):
        asyncio.run(d.pull(h, {"w": fake_dest(torch.int8)}, channel_scales={"w": scale_for("channel")}))
    with pytest.raises(ValueError, match="does not apply to int8 destinations"):
        asyncio.run(d.pull(h, {"w": fake_dest(torch.int8)}, channel_scales={"w": scale_for("channel")}, verbatim=True,
                           scale_fmt="ue8m0"))
    with pytest.raises(ValueError, match="mix scaled int8 and scaled fp8"):
        asyncio.run(d.pull({"w": [scaled_handle(torch.int8, "channel"), scaled_handle(E4M3, "channel")]},
                           {"w": torch.zeros(4, 4)}))
    assert d._plan is None


# ---- plans -----------------------------------------------------------------------------------------------------------
def test_int8_dequant_names_get_their_own_plan(monkeypatch):
    from torchstore_b200 import direct_weight_sync as dws

    seen = []
    monkeypatch.setattr(dws.Plans, "build", classmethod(lambda cls, per_device: dws.Plans()))
    monkeypatch.setattr(dws.Plans, "build_dequant_fp8", classmethod(
        lambda cls, per_device: seen.append({dev: [type(s).__name__ for s in args[1]] for dev, args in per_device.items()})
        or {0: len(seen)}))
    monkeypatch.setattr(DirectWeightSyncDest, "op_windows", staticmethod(lambda op, w: (w, w)))
    monkeypatch.setattr(dws, "_add_dq_source", lambda sources, op, dev: sources.setdefault(id(op.rdma_buffer),
                                                                                           (op.name, object())))

    class Buf(dws.NvlinkBuffer):
        def __init__(self, dtype):
            self._dtype = dtype

        dtype = property(lambda self: self._dtype)

        def window(self, dev):
            return None

    dest = types.SimpleNamespace(is_cuda=True, device=torch.device("cuda", 0))
    d = DirectWeightSyncDest()
    d._plan = [types.SimpleNamespace(name=n, dest_local=dest, rdma_buffer=Buf(dt))
               for n, dt in (("f", E4M3), ("i", torch.int8), ("j", torch.int8))]
    d._compile({}, {"f", "i", "j"})
    assert len(seen) == 2 and d._dequant_plans == {0: 1} and d._int8_dequant_plans == {0: 2}
    assert any(p is d._int8_dequant_plans for p in d._fp8_plans)


@pytest.mark.parametrize("built,now", [(E4M3, torch.int8), (torch.int8, E4M3)])
def test_plan_rebuilds_on_a_dtype_flip(monkeypatch, built, now):
    """A verbatim pull's cached plan is dropped when a scaled name's destination changes between float8_e4m3fn and
    int8 at the same address (with handles of the matching format), and kept while it does not."""
    plans_built = []
    monkeypatch.setattr(DirectWeightSyncDest, "_build_plan", lambda self, *a, **k: plans_built.append(1) or [])
    monkeypatch.setattr(DirectWeightSyncDest, "_verbatim_rects", staticmethod(lambda plan, scaled: {}))
    monkeypatch.setattr(DirectWeightSyncDest, "_compile", lambda self, *a, **k: None)
    scales = {"w": scale_for("channel")}
    d = DirectWeightSyncDest()
    for dtype, n in ((built, 1), (built, 1), (now, 2), (now, 2)):
        asyncio.run(d.pull({"w": [scaled_handle(dtype, "channel")]}, {"w": fake_dest(dtype)}, channel_scales=scales,
                           verbatim=True))
        assert len(plans_built) == n
    d.close()

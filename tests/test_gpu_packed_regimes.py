"""The packed-destination regimes (tests/packed_regimes.py) on the GPU: every regime, route and variant pulled by
``DirectWeightSyncDest.pull`` from handles on cuda:0 and compared bit for bit with the numpy reference (bytes and
scales, sentinels outside every part untouched); random specs with special values at part and group boundaries;
``transfer_dtype`` staging; the requantised Qwen3 TP8 w13 block that straddles two parts against the reference;
a grouped pull refused for a hole and the same puller pulling the corrected spec; and parts landing past byte 2^32 of
their destination."""

import numpy as np
import pytest
import torch

from oracle import block_fp8_oracle, dequant_fp8_oracle, packed_oracle
from tests import packed_regimes as pr
from tests.helpers import DEV, needs_two_gpus, run
from torchstore_b200.direct_weight_sync import (DirectWeightSyncDest, DirectWeightSyncSource, NvlinkBuffer, PackedPart,
                                                RDMAWeightHandle, ScaledNvlinkBuffer, source_scale_shapes)
from torchstore_b200.transport.types import TensorSlice

pytestmark = pytest.mark.gpu


def make_buffer(device):
    def make(shard, scale, g, r0, c0):
        if g is None:
            return NvlinkBuffer(shard.to(device))
        return ScaledNvlinkBuffer(shard.to(device), scale.to(device), g, r0, c0)
    return make


def device_pull(spec, data, sync=None, device=DEV):
    """Pull ``spec`` into fresh sentinel-filled destinations on cuda:0 -> (result, sync, handles)."""
    handles = pr.handles_of(spec, data, make_buffer(device))
    dests, scales, slices = pr.dests_of(spec, DEV)
    sync = sync or DirectWeightSyncDest()
    run(sync.pull(handles, dests, slices or None, packed=spec.packed(), **spec.kw(), **{k: v or None for k, v in scales.items()}))
    return dests, scales, handles, sync


def result(dests, scales):
    return {n: (d, next((s[n] for s in scales.values() if n in s), None)) for n, d in dests.items()}


@pytest.mark.parametrize("variant", pr.VARIANTS)
@pytest.mark.parametrize("regime,route", pr.CASES, ids=[f"{r}-{ro}" for r, ro in pr.CASES])
def test_regime_on_the_device(regime, route, variant, monkeypatch):
    builds = []
    orig = DirectWeightSyncDest._build_plan
    monkeypatch.setattr(DirectWeightSyncDest, "_build_plan", lambda self, *a, **k: builds.append(1) or orig(self, *a, **k))
    spec = pr.spec(regime, route)
    data = pr.make_data(spec, 11, special=variant == "special")
    dests, scales, handles, sync = device_pull(spec, data)
    pr.assert_pull(spec, result(dests, scales), pr.expect(spec, data), f"{regime}/{route}/{variant}")
    if variant == "update":
        # new source values in the same memory: the second pull gives them, from the plan of the first
        new = pr.make_data(spec, 1011)
        pr.refill(spec, handles, new, lambda b: b._keepalive, lambda b: b._scale_keepalive)
        torch.cuda.synchronize()
        run(sync.pull(handles, dests, pr.dests_of(spec)[2] or None, packed=spec.packed(), **spec.kw(),
                      **{k: v or None for k, v in scales.items()}))
        pr.assert_pull(spec, result(dests, scales), pr.expect(spec, new), f"{regime}/{route}/update")
    assert len(builds) == 1
    sync.close()


@pytest.mark.parametrize("chunk", range(4))
def test_random_specs_on_the_device(chunk):
    """Random specs with special values planted at part boundaries and group edges (every other seed)."""
    for seed in range(1000 + 12 * chunk, 1000 + 12 * (chunk + 1)):
        spec = pr.random_spec(seed)
        data = pr.make_data(spec, seed, special=seed % 2 == 0)
        if pr.refusal(spec):
            with pytest.raises(ValueError, match=pr.refusal(spec)):
                device_pull(spec, data)
            continue
        dests, scales, _, sync = device_pull(spec, data)
        pr.assert_pull(spec, result(dests, scales), pr.expect(spec, data), f"random spec {seed}")
        sync.close()


STAGING = [("row_parts_unaligned", "bfloat16", "e4m3"), ("col_parts", "float32", "bfloat16"),
           ("drop_two_lead", "bfloat16", "e5m2"), ("sharded_sources", "float16", "float32")]


@pytest.mark.parametrize("regime,src,staging", STAGING)
def test_transfer_dtype_staging(regime, src, staging):
    """Sources registered with ``transfer_dtype`` (the refresh casts into staging) pulled as bytes into packed
    destinations of the staging dtype: each part holds its source converted as the fp8 oracle converts it."""
    r = pr.REGIMES[regime]
    spec = pr.Spec({n: pr.Src(shape, src, None, boxes) for n, (shape, boxes) in r.sources.items()},
                   {"w": pr.Dst(r.shape, staging, parts=r.parts)})
    data = pr.make_data(spec, 5, special=True)
    handles, srcs = {}, []
    for name, s in spec.sources.items():
        for k, (off, loc) in enumerate(s.boxes):
            src_ = DirectWeightSyncSource()
            local = data.full[name][tuple(slice(o, o + e) for o, e in zip(off, loc))].contiguous().to(DEV)
            h = src_.register({name: local}, rank=k, transfer_dtype=pr.DT[staging],
                              tensor_slices={name: TensorSlice(off, (k,), s.shape, loc, (len(s.boxes),))})[name]
            handles.setdefault(name, []).append(h)
            srcs.append(src_)
    dests, _, _ = pr.dests_of(spec, DEV)
    sync = DirectWeightSyncDest()
    run(sync.pull(handles, dests, packed=spec.packed()))
    want = pr.expect(pr.Spec({n: pr.Src(s.shape, staging, None, s.boxes) for n, s in spec.sources.items()}, spec.dests),
                     pr.Data({n: pr.convert(x, src, staging) for n, x in data.full.items()}))
    pr.assert_pull(spec, result(dests, {}), want, f"{regime} staged {src} -> {staging}")
    sync.close()


@pytest.mark.parametrize("route", ["dq_e4m3_block_bfloat16", "dq_int8_tensor_float16", "rq_channel_block"])
def test_scaled_sources_into_a_dropped_column_dim_are_refused_then_a_quantising_pull_takes_it(route):
    """dest[R, C, 2] at [..., k] from scaled handles is refused before anything is compiled, naming the destination
    and the part; the same puller then quantises the same parts from bf16 handles."""
    r, ro = pr.REGIMES["drop_col_dim"], pr.ROUTES[route]
    spec = pr.Spec({n: pr.Src(shape, ro.src, ro.sg, boxes) for n, (shape, boxes) in r.sources.items()},
                   {"w": pr.Dst(r.shape, ro.out, ro.g, r.parts)}, requantize=ro.kind == "requant")
    sync = DirectWeightSyncDest()
    with pytest.raises(ValueError, match=pr.refusal(spec)):
        device_pull(spec, pr.make_data(spec, 6), sync)
    assert sync._plan is None and not any(sync._fp8_plans) and not sync._native_plans
    ok = pr.spec("drop_col_dim", "quant_fp8_block_bfloat16")
    data = pr.make_data(ok, 6, special=True)
    dests, scales, _, _ = device_pull(ok, data, sync)
    pr.assert_pull(ok, result(dests, scales), pr.expect(ok, data), "drop_col_dim after the refusal")
    sync.close()


def test_qwen3_tp8_w13_straddling_block_requantised_to_the_reference():
    """Qwen3-30B-A3B's w13 at TP8 holds 96-row gate and up halves: verbatim is refused for block row 0, which
    straddles both parts, and the requantising pull writes the reference's bytes and scales for every block."""
    full = {n: (torch.randn(768, 256, generator=torch.Generator().manual_seed(53 + i)) * 0.02).to(torch.bfloat16)
            for i, n in enumerate(("gate", "up"))}
    src = DirectWeightSyncSource()
    handles = {n: [h] for n, h in src.register({n: t.to(DEV) for n, t in full.items()}, rank=0,
                                                quantize={"gate": "block", "up": "block"}).items()}
    parts = (PackedPart("gate", (0, slice(0, 96), slice(0, 256)), (96, 0)),
             PackedPart("up", (0, slice(96, 192), slice(0, 256)), (96, 0)))
    q = torch.zeros(1, 192, 256, dtype=pr.E4M3, device=DEV)
    s = torch.full(source_scale_shapes("block", (1, 192, 256), 0, 0)[0], -1.0, device=DEV)
    sync = DirectWeightSyncDest()
    with pytest.raises(ValueError, match=r"verbatim pull of 'w13' \(block_scales\): destination block \(0, 0, 0\)"):
        run(sync.pull(handles, {"w13": q}, packed={"w13": parts}, block_scales={"w13": s}, verbatim=True))
    assert sync._plan is None
    run(sync.pull(handles, {"w13": q}, packed={"w13": parts}, block_scales={"w13": s}, requantize=True))
    x = {}
    for n, (qb, sb, _) in src._quantized.items():
        bits = dequant_fp8_oracle.dequantize(qb.view(torch.uint8).cpu().numpy(), sb.cpu().numpy(), "block", 0, 0, "float32")
        x[n] = bits.view(np.float32)
    want_q, want_s = block_fp8_oracle.quantize(packed_oracle.fill(np.zeros((1, 192, 256), np.float32), parts, x))
    assert np.array_equal(q.view(torch.uint8).cpu().numpy(), want_q)
    assert np.array_equal(s.cpu().numpy().view(np.uint32), want_s.view(np.uint32))
    assert s.shape == (1, 2, 2) and (s > 0).all()
    sync.close()


@pytest.mark.parametrize("route", ["quant_fp8_block_bfloat16", "quant_int8_channel_bfloat16", "rq_block_block"])
def test_grouped_pull_with_a_hole_is_refused_then_the_corrected_spec_pulls(route):
    r, ro = pr.REGIMES["holes"], pr.ROUTES[route]
    srcs = {n: pr.Src(shape, ro.src, ro.sg, boxes) for n, (shape, boxes) in r.sources.items()}
    holed = pr.Spec(srcs, {"w": pr.Dst(r.shape, ro.out, ro.g, r.parts)}, requantize=ro.kind == "requant")
    data = pr.make_data(holed, 8)
    handles = pr.handles_of(holed, data, make_buffer(DEV))
    dests, scales, _ = pr.dests_of(holed, DEV)
    sync = DirectWeightSyncDest()
    with pytest.raises(ValueError, match=r"pull of 'w' \(\w+_scales\): .*target 0"):
        run(sync.pull(handles, dests, packed=holed.packed(), requantize=holed.requantize,
                      **{k: v or None for k, v in scales.items()}))
    assert sync._plan is None
    # the same puller, the same handles: parts that cover the destination
    full = (PackedPart("a", (slice(0, 30), slice(0, 150)), (0, 3)), PackedPart("b", (slice(0, 30), slice(150, 200)), (0, 0)),
            PackedPart("b", (slice(30, 64), slice(10, 200)), (0, 0)), PackedPart("b", (slice(30, 64), slice(0, 10)), (6, 180)))
    fixed = pr.Spec(srcs, {"w": pr.Dst(r.shape, ro.out, ro.g, full)}, requantize=holed.requantize)
    run(sync.pull(handles, dests, packed=fixed.packed(), requantize=fixed.requantize,
                  **{k: v or None for k, v in scales.items()}))
    pr.assert_pull(fixed, result(dests, scales), pr.expect(fixed, data), f"holes/{route} corrected")
    sync.close()


# ---- past byte 2^32 -----------------------------------------------------------------------------------------------
def test_byte_copy_part_past_4_gib():
    """A bf16 destination of [32832, 65536] (4.008 GiB) whose part box starts at row 32769, column 3: byte
    2^32 + 131078.  The 8 MiB source reads from (1, 2).  About 4.6 GB of device memory at the peak (the destination,
    plus 0.5 GB of the sentinel check's row chunks)."""
    rows, cols = 32832, 65536
    dest = torch.full((rows, cols), -3, dtype=torch.int16, device=DEV).view(torch.bfloat16)
    src = (torch.randn(64, cols, device=DEV) * 0.02).to(torch.bfloat16)
    z = (0, 0)
    handles = {"s": [RDMAWeightHandle(NvlinkBuffer(src), TensorSlice(z, (0,), (64, cols), (64, cols), (1,)), 0)]}
    part = PackedPart("s", (slice(32769, 32829), slice(3, 65000)), (1, 2))
    assert (32769 * cols + 3) * 2 > 2 ** 32
    sync = DirectWeightSyncDest()
    run(sync.pull(handles, {"w": dest}, packed={"w": (part,)}))
    torch.cuda.synchronize()
    window = dest[32760:32832].view(torch.int16).cpu().numpy()
    want = packed_oracle.fill(np.full((72, cols), -3, np.int16),
                              (PackedPart("s", (slice(9, 69), slice(3, 65000)), (1, 2)),),
                              {"s": src.view(torch.int16).cpu().numpy()})
    assert np.array_equal(window, want)
    for r in range(0, 32760, 4095):  # rows before the part keep their sentinel, in 0.5 GB chunks
        assert bool((dest[r:min(r + 4095, 32760)].view(torch.int16) == -3).all()), r
    sync.close()
    del dest, src
    torch.cuda.empty_cache()


def test_block_quantising_part_past_4_gib():
    """A block-scaled e4m3 destination of [33024, 131072] (4.03 GiB): four parts of 8192 rows read one 2 GiB bf16
    source [8192, 131072], and the last 256 rows come from a 64 MiB source [400, 131072] as two parts, the second's
    box starting at row 32770 (byte 2^32 + 262144) and reading from source row 99, off the source's blocks.  About
    6.6 GB (6.13 GiB) of device memory.  The blocks past byte 2^32 and the first block row equal the reference."""
    rows, cols = 33024, 131072
    a = (torch.randn(8192, cols, device=DEV) * 0.05).to(torch.bfloat16)
    b = (torch.randn(400, cols, device=DEV) * 0.05).to(torch.bfloat16)
    z = (0, 0)
    handles = {"a": [RDMAWeightHandle(NvlinkBuffer(a), TensorSlice(z, (0,), tuple(a.shape), tuple(a.shape), (1,)), 0)],
               "b": [RDMAWeightHandle(NvlinkBuffer(b), TensorSlice(z, (0,), tuple(b.shape), tuple(b.shape), (1,)), 0)]}
    parts = tuple(PackedPart("a", (slice(8192 * i, 8192 * (i + 1)), slice(0, cols)), (0, 0)) for i in range(4)) + (
        PackedPart("b", (slice(32768, 32770), slice(0, cols)), (7, 0)),
        PackedPart("b", (slice(32770, 33024), slice(0, cols)), (99, 0)))
    assert 32770 * cols > 2 ** 32
    q = torch.zeros(rows, cols, dtype=pr.E4M3, device=DEV)
    s = torch.full(source_scale_shapes("block", (rows, cols), 0, 0)[0], -1.0, device=DEV)
    sync = DirectWeightSyncDest()
    run(sync.pull(handles, {"w": q}, packed={"w": parts}, block_scales={"w": s}))
    torch.cuda.synchronize()
    tail = np.zeros((256, cols), np.float32)
    tail[:2], tail[2:] = b[7:9].float().cpu().numpy(), b[99:353].float().cpu().numpy()
    want_q, want_s = block_fp8_oracle.quantize(tail)
    assert np.array_equal(q[32768:].view(torch.uint8).cpu().numpy(), want_q)
    assert np.array_equal(s[256:].cpu().numpy().view(np.uint32), want_s.view(np.uint32))
    head_q, head_s = block_fp8_oracle.quantize(a[:128].float().cpu().numpy())
    assert np.array_equal(q[:128].view(torch.uint8).cpu().numpy(), head_q)
    assert np.array_equal(s[:1].cpu().numpy().view(np.uint32), head_s.view(np.uint32))
    sync.close()
    del a, b, q, s
    torch.cuda.empty_cache()


# ---- peer handles ---------------------------------------------------------------------------------------------------
@needs_two_gpus
@pytest.mark.parametrize("route", ["copy_bf16", "quant_fp8_block_bfloat16", "dq_e4m3_block_bfloat16"])
def test_sharded_sources_on_a_peer(route):
    """sharded_sources with every handle on cuda:1, read over the peer mapping by cuda:0's plans."""
    spec = pr.spec("sharded_sources", route)
    data = pr.make_data(spec, 21, special=True)
    dests, scales, _, sync = device_pull(spec, data, device="cuda:1")
    pr.assert_pull(spec, result(dests, scales), pr.expect(spec, data), f"sharded_sources/{route} on cuda:1")
    sync.close()

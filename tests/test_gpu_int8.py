"""Scaled INT8 destinations on the H100: bf16/f16/f32 handles quantised into block-, channel- and tensor-scaled int8
during the pull, bit for bit against the numpy oracle (int8 bytes and scale_inv bits); reshards, MoE stacks,
partial edge blocks, the two-pass paths, NaN / Inf / zero groups, mixed pulls, replays, the state-dict API, the
refusals, FSDP -> TP over peer mappings (two GPUs), and the full-size Llama-3-8B linear weights against the
torch-CUDA rendering.  Several "ranks" are emulated as several sources on cuda:0."""

import numpy as np
import pytest
import torch

from oracle.int8_oracle import (GRANULARITIES, SPECIALS, bits_of, quantize, same_scales, scale_shape, special_stack,
                                synth_f32, torch_quantize, widen)
from tests.fp8_regimes import whole
from tests.helpers import DEV, E4M3, I8, KW, cleanup, needs_two_gpus, pull_box, run
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource
from torchstore_b200.transport.types import TensorSlice

pytestmark = pytest.mark.gpu
DTYPES = (torch.bfloat16, torch.float16, torch.float32)


def publish(full: torch.Tensor, boxes, name="w", device=DEV, **register_kw):
    """One source per box (offsets, extents) of `full`, registered on `device` -> (sources, handles)."""
    sources, handles = [], []
    for r, (off, loc) in enumerate(boxes):
        shard = full[tuple(slice(o, o + e) for o, e in zip(off, loc))].contiguous().to(device)
        ts = TensorSlice(tuple(off), (r,), tuple(full.shape), tuple(loc), (len(boxes),))
        src = DirectWeightSyncSource()
        handles.append(src.register({name: shard}, rank=r, tensor_slices={name: ts}, **register_kw)[name])
        sources.append((src, shard))
    return sources, handles


def rows(shape, k):
    n = shape[-2]
    cuts = [i * n // k for i in range(k)] + [n]
    lead = tuple(0 for _ in shape[:-2])
    return [(lead + (a, 0), tuple(shape[:-2]) + (b - a, shape[-1])) for a, b in zip(cuts, cuts[1:])]


def cols(shape, cuts):
    lead = tuple(0 for _ in shape[:-2])
    edges = [0] + list(cuts) + [shape[-1]]
    return [(lead + (0, a), tuple(shape[:-1]) + (b - a,)) for a, b in zip(edges, edges[1:])]


def int8_dest(g, shape, device=DEV):
    q = torch.full(shape, 0x55, dtype=torch.int8, device=device)
    return q, torch.full(scale_shape(g, shape), -1.0, device=device)


def assert_exact(q, s, x, g):
    """Bit-exact with the numpy oracle: int8 bytes, and scale_inv bits (NaN-agnostic for NaN scales)."""
    want_q, want_s = quantize(widen(bits_of(x.cpu()), str(x.dtype)[6:]), g)
    assert np.array_equal(q.cpu().numpy(), want_q)
    assert same_scales(s.cpu().numpy().reshape(want_s.shape), want_s)


LAYOUTS = {
    "exact_300x520": ((300, 520), lambda s: [((0, 0), s)]),
    "fsdp4_rows_ragged_300x200": ((300, 200), lambda s: rows(s, 4)),
    "fsdp4_cols": ((256, 512), lambda s: cols(s, (128, 256, 384))),
    "unaligned_cols_at_70_and_201": ((260, 330), lambda s: cols(s, (70, 201))),
    "moe_3x130x260": ((3, 130, 260), lambda s: [((0, 0, 0), s)]),
    "moe_rows_3x130x260": ((3, 130, 260), lambda s: rows(s, 2)),
}


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("g", GRANULARITIES)
def test_quantising_pull_is_exact(g, dtype, layout):
    shape, boxes = LAYOUTS[layout]
    full = synth_f32(shape, 201 + len(layout)).to(dtype)
    sources, handles = publish(full, boxes(shape))
    sync, q, s, _ = pull_box(handles, shape, whole(shape), I8, granularity=g)
    sync.close()
    assert_exact(q, s, full, g)
    cleanup(sources)


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
def test_long_channel_rows_and_tensors_take_the_two_pass_path(dtype):
    shape = (3, 16400 if dtype != torch.float32 else 8200)  # rows over the 32 KiB stage
    full = synth_f32(shape, 7).to(dtype)
    sources, handles = publish(full, cols(shape, (shape[1] // 2,)))
    for g in ("channel", "tensor"):
        sync, q, s, _ = pull_box(handles, shape, whole(shape), I8, granularity=g)
        sync.close()
        assert_exact(q, s, full, g)
    cleanup(sources)


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("g", GRANULARITIES)
def test_nan_inf_zero_ties_max_and_subnormal_groups(g, dtype):
    """The special stack of the fixture: NaN, Inf and NaN+Inf groups give q = 0 with NaN / Inf scale_inv, a zero
    group the 1e-4 floor, ties round half to even."""
    full = special_stack(dtype)
    shape = tuple(full.shape)
    sources, handles = publish(full, rows(shape, 2))
    sync, q, s, _ = pull_box(handles, shape, whole(shape), I8, granularity=g)
    sync.close()
    assert_exact(q, s, full, g)
    qc, sc = q.cpu(), s.cpu()
    for k, kind in enumerate(SPECIALS):
        if kind in ("nan", "inf", "nan_inf"):
            assert (qc[k] == 0).all() and (torch.isinf(sc[k]) if kind == "inf" else torch.isnan(sc[k])).all()
    cleanup(sources)


def test_mixed_pull_of_fp8_int8_and_plain_names():
    shape = (384, 256)
    names = {"fb": ("block", E4M3), "ib": ("block", torch.int8), "ic": ("channel", torch.int8),
             "ft": ("tensor", E4M3), "it": ("tensor", torch.int8), "plain": (None, torch.bfloat16),
             "bytes": (None, torch.int8)}
    fulls = {n: synth_f32(shape, 40 + i).to(torch.bfloat16) for i, n in enumerate(names)}
    fulls["bytes"] = torch.randint(-128, 128, shape, dtype=torch.int8)
    handles, sources = {}, []
    for n, full in fulls.items():
        s, h = publish(full, rows(shape, 2), name=n)
        sources += s
        handles[n] = h
    dests, scales = {}, {kw: {} for kw in KW.values()}
    for n, (g, dt) in names.items():
        dests[n] = torch.zeros(shape, dtype=dt, device=DEV)
        if g:
            scales[KW[g]][n] = torch.full(scale_shape(g, shape), -1.0, device=DEV)
    d = DirectWeightSyncDest()
    run(d.pull(handles, dests, **scales))
    for n, (g, dt) in names.items():
        if dt == torch.int8 and g:
            assert_exact(dests[n], scales[KW[g]][n], fulls[n], g)
        elif g:
            from oracle.ue8m0_oracle import torch_quantize as fp8_quantize

            tq, ts = fp8_quantize(fulls[n].to(DEV), g)
            assert torch.equal(dests[n].view(torch.uint8), tq.view(torch.uint8))
            assert torch.equal(scales[KW[g]][n].view(torch.int32), ts.reshape(scales[KW[g]][n].shape).view(torch.int32))
        else:
            assert torch.equal(dests[n].cpu(), fulls[n])
    assert d._int8_block_plans and d._int8_scaled_plans and d._block_plans and d._scaled_plans
    d.close()
    cleanup(sources)


def test_replay_after_the_source_weights_change_and_dtype_flip():
    shape = (256, 384)
    full = synth_f32(shape, 3).to(torch.bfloat16)
    sources, handles = publish(full, rows(shape, 2))
    q, s = int8_dest("channel", shape)
    d = DirectWeightSyncDest()
    run(d.pull({"w": handles}, {"w": q}, channel_scales={"w": s}))
    assert_exact(q, s, full, "channel")
    full2 = synth_f32(shape, 4).to(torch.bfloat16) * 3
    for (_, shard), (off, loc) in zip(sources, rows(shape, 2)):
        shard.copy_(full2[off[0]: off[0] + loc[0]].to(DEV))
    run(d.pull({"w": handles}, {"w": q}, channel_scales={"w": s}))  # cached plan, new values
    assert_exact(q, s, full2, "channel")
    f8 = torch.zeros(shape, dtype=E4M3, device=DEV)
    run(d.pull({"w": handles}, {"w": f8}, channel_scales={"w": s}))  # an fp8 destination: rebuilt
    from oracle.ue8m0_oracle import torch_quantize as fp8_quantize

    tq, _ = fp8_quantize(full2.to(DEV), "channel")
    assert torch.equal(f8.view(torch.uint8), tq.view(torch.uint8)) and not d._int8_scaled_plans
    d.close()
    cleanup(sources)


def test_state_dict_api():
    import torch.distributed as dist
    from torch.testing._internal.distributed.fake_pg import FakeStore

    import torchstore_b200 as ts

    async def main():
        dist.init_process_group("fake", store=FakeStore(), rank=0, world_size=1)
        await ts.initialize()
        try:
            src = {"a": synth_f32((256, 384), 61).to(torch.bfloat16).to(DEV),
                   "b": synth_f32((2, 64, 300), 62).to(torch.float16).to(DEV)}
            await ts.put_state_dict(src, "policy_i8", direct_rdma=True)
            dst = {"a": torch.zeros(256, 384, dtype=torch.int8, device=DEV), "b": torch.zeros(2, 64, 300, dtype=torch.int8, device=DEV)}
            bs, tsc = {"a": torch.zeros(2, 3, device=DEV)}, {"b": torch.zeros(2, device=DEV)}
            for _ in range(2):
                out = await ts.get_state_dict("policy_i8", user_state_dict=dst, direct_rdma=True, block_scales=bs,
                                              tensor_scales=tsc)
                assert out is dst
                assert_exact(dst["a"], bs["a"], src["a"], "block")
                assert_exact(dst["b"], tsc["b"], src["b"], "tensor")
                src["a"].mul_(0.5)
                src["b"].mul_(3.0)
                await ts.put_state_dict(None, "policy_i8", direct_rdma=True)
        finally:
            await ts.shutdown()
            dist.destroy_process_group()

    run(main())


def test_refusals_on_the_device():
    shape = (128, 256)
    full = synth_f32(shape, 5)
    q8 = full.to(DEV).to(E4M3)
    s = torch.full((1, 2), 0.01, device=DEV)
    src = DirectWeightSyncSource()
    h = src.register({"w": q8}, rank=0, block_scales={"w": s})["w"]
    for kw in ({}, {"requantize": True}, {"verbatim": True}):
        qi, si = int8_dest("block", shape)
        with pytest.raises(TypeError, match="int8 destinations are quantised from bf16, f16 or f32 handles"):
            run(DirectWeightSyncDest().pull({"w": [h]}, {"w": qi}, block_scales={"w": si}, **kw))
    run(src.cleanup())
    sources, handles = publish(full.to(torch.bfloat16), [((0, 0), shape)])
    qi, si = int8_dest("channel", shape)
    with pytest.raises(ValueError, match="does not apply to int8"):
        run(DirectWeightSyncDest().pull({"w": handles}, {"w": qi}, channel_scales={"w": si}, scale_fmt="ue8m0"))
    with pytest.raises(NotImplementedError, match="no fused cast kernel"):  # unscaled int8: a byte move, as before
        run(DirectWeightSyncDest().pull({"w": handles}, {"w": qi}))
    cleanup(sources)


@needs_two_gpus
@pytest.mark.parametrize("g", GRANULARITIES)
def test_fsdp_to_tp_over_peer_mappings(g):
    """FSDP(2) row shards on cuda:0 and cuda:1 pulled into TP(2) column shards on both devices."""
    shape = (512, 768)
    full = synth_f32(shape, 77).to(torch.bfloat16)
    sources, handles = [], []
    for r, (off, loc) in enumerate(rows(shape, 2)):
        s, h = publish(full, [(off, loc)], device=f"cuda:{r}")
        sources += s
        handles += h
    for t in range(2):
        dev = f"cuda:{t}"
        c0, c1 = t * 384, (t + 1) * 384
        q, s = int8_dest(g, (512, 384), device=dev)
        ts = TensorSlice((0, c0), (t,), shape, (512, 384), (2,))
        d = DirectWeightSyncDest()
        run(d.pull({"w": handles}, {"w": q}, {"w": ts}, **{KW[g]: {"w": s}}))
        assert_exact(q, s, full[:, c0:c1], g)
        d.close()
    cleanup(sources)


LLAMA3_8B = {"wq": (4096, 4096), "wk": (1024, 4096), "wv": (1024, 4096), "wo": (4096, 4096), "w1": (14336, 4096),
             "w2": (4096, 14336), "w3": (14336, 4096)}


def test_llama3_8b_linear_weights_per_channel_full_size():
    fulls = {n: (torch.randn(shape, device=DEV) * 0.02).to(torch.bfloat16) for n, shape in LLAMA3_8B.items()}
    src = DirectWeightSyncSource()
    handles = src.register(fulls, rank=0)
    dests = {n: torch.zeros(shape, dtype=torch.int8, device=DEV) for n, shape in LLAMA3_8B.items()}
    scales = {n: torch.zeros(shape[0], 1, device=DEV) for n, shape in LLAMA3_8B.items()}
    d = DirectWeightSyncDest()
    run(d.pull({n: [h] for n, h in handles.items()}, dests, channel_scales=scales))
    for n in LLAMA3_8B:
        tq, ts = torch_quantize(fulls[n], "channel")
        assert torch.equal(dests[n], tq), n
        assert torch.equal(scales[n].view(torch.int32), ts.view(torch.int32)), n
    d.close()
    run(src.cleanup())

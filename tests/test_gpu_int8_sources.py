"""Scaled INT8 sources on the H100: source-side int8 quantisation (``register(quantize=..., quant_dtype=torch.int8)``)
bit for bit against the torch-CUDA rendering and the numpy oracle (int8 bytes, scale_inv bits) on FSDP-style shards
with mid-block boundaries, MoE stacks, the two-pass paths, NaN / Inf / zero / tie groups and refresh(); int8
checkpoints dequantised into bf16/f16/f32 across reshards; verbatim int8 chains; a mixed pull; the state-dict API;
peer mappings (two GPUs); and the full-size Llama-3-8B linear weights, FSDP(8) -> TP(8), with the two cross-checks
that need no oracle: source-side int8 + verbatim pull equals the destination-side int8 quantising pull wherever
the groups coincide, and source-side int8 of an unsharded tensor equals the destination-side pull from it.  Several
"ranks" are emulated as several sources on cuda:0."""

import numpy as np
import pytest
import torch

from oracle.int8_oracle import SPECIALS, same_scales, special_stack
from oracle.int8_source_oracle import (GRANULARITIES, bits_of, int8_of, quantize, scale_of, scale_shape, synth_f32,
                                       torch_dequantize, torch_quantize, widen)
from tests.helpers import DEV, E4M3, I8, KW, cleanup, needs_two_gpus, register_boxes, register_shards, run
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource
from torchstore_b200.transport.types import TensorSlice

pytestmark = pytest.mark.gpu
DTYPES = (torch.bfloat16, torch.float16, torch.float32)


def rows(shape, cuts):
    lead = tuple(0 for _ in shape[:-2])
    edges = [0] + list(cuts) + [shape[-2]]
    return [(lead + (a, 0), tuple(shape[:-2]) + (b - a, shape[-1])) for a, b in zip(edges, edges[1:])]


def cols(shape, cuts):
    lead = tuple(0 for _ in shape[:-2])
    edges = [0] + list(cuts) + [shape[-1]]
    return [(lead + (0, a), tuple(shape[:-1]) + (b - a,)) for a, b in zip(edges, edges[1:])]


def box(full, off, loc):
    return full[tuple(slice(o, o + e) for o, e in zip(off, loc))]


def staging(src, name="w"):
    q, s, _ = src._quantized[name]
    return q, s


def assert_staging_exact(src, shard, g, r0, c0, name="w"):
    """The staging of one source against the torch-CUDA rendering (bytes, scale bits) and the numpy oracle."""
    q, s = staging(src, name)
    assert q.dtype == torch.int8
    tq, ts = torch_quantize(shard, g, r0, c0)
    assert torch.equal(q, tq)
    assert same_scales(s.cpu().numpy(), ts.reshape(s.shape).cpu().numpy())
    want_q, want_s = quantize(widen(bits_of(shard.cpu()), str(shard.dtype)[6:]), g, r0, c0)
    assert np.array_equal(q.cpu().numpy(), want_q) and same_scales(s.cpu().numpy(), want_s)


LAYOUTS = {  # shape, boxes: FSDP row shards cut mid-block, unaligned column shards, MoE stacks
    "whole_300x520": ((300, 520), lambda s: [((0, 0), s)]),
    "fsdp_rows_mid_block_300x200": ((300, 200), lambda s: rows(s, (75, 150, 225))),
    "cols_at_70_and_201": ((260, 330), lambda s: cols(s, (70, 201))),
    "moe_rows_3x130x260": ((3, 130, 260), lambda s: rows(s, (37,))),
}


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("g", GRANULARITIES)
def test_source_side_int8_is_exact(g, dtype, layout):
    shape, boxes = LAYOUTS[layout]
    full = synth_f32(shape, 301 + len(layout)).to(dtype)
    sources, handles = register_boxes(full, boxes(shape), quantize={"w": g}, quant_dtype=I8)
    for (src, shard, _), (off, _) in zip(sources, boxes(shape)):
        assert_staging_exact(src, shard, g, off[-2], off[-1])
        assert src._handles["w"].rdma_buffer.dtype == torch.int8
    cleanup(sources)


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("g", GRANULARITIES)
def test_nan_inf_zero_and_tie_groups(g, dtype):
    full = special_stack(dtype)
    sources, _ = register_boxes(full, [((0, 0, 0), tuple(full.shape))], quantize={"w": g}, quant_dtype=I8)
    src, shard, _ = sources[0]
    assert_staging_exact(src, shard, g, 0, 0)
    q, s = staging(src)
    for k, kind in enumerate(SPECIALS):
        if kind in ("nan", "inf", "nan_inf"):
            assert (q[k] == 0).all() and (torch.isinf(s[k]) if kind == "inf" else torch.isnan(s[k])).all()
    cleanup(sources)


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
def test_two_pass_paths(dtype):
    shape = (3, 16400 if dtype != torch.float32 else 8200)  # rows over the 32 KiB stage
    full = synth_f32(shape, 9).to(dtype)
    for g in ("channel", "tensor"):
        sources, _ = register_boxes(full, rows(shape, (1,)), quantize={"w": g}, quant_dtype=I8)
        for (src, shard, _), off in zip(sources, (0, 1)):
            assert_staging_exact(src, shard, g, off, 0)
        cleanup(sources)


def test_refresh_after_the_weights_change():
    shape = (300, 260)
    full = synth_f32(shape, 12).to(torch.bfloat16)
    for g in GRANULARITIES:
        sources, _ = register_boxes(full, rows(shape, (100,)), quantize={"w": g}, quant_dtype=I8)
        for k in range(2):
            for _, shard, _ in sources:
                shard.mul_(3.0 if k else 0.25)
            for src, *_ in sources:
                assert src.refresh() == 1
            for (src, shard, _), r0 in zip(sources, (0, 100)):
                assert_staging_exact(src, shard, g, r0, 0)
        cleanup(sources)


@pytest.mark.parametrize("dst", DTYPES, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("g", GRANULARITIES)
def test_int8_checkpoints_dequantise_across_reshards(g, dst):
    """FSDP-style row shards of an int8 checkpoint (each with its shard-local scale) pulled into TP column shards of
    a bf16/f16/f32 model: each element is (q.float() * scale).to(dst) of the shard it is read from."""
    shape = (2, 300, 520)
    q = int8_of(shape, 21)
    boxes = rows(shape, (75, 200))
    scales = [scale_of(scale_shape(g, loc, off[-2], off[-1]), 30 + i) for i, (off, loc) in enumerate(boxes)]
    shards = [(off, box(q, off, loc).contiguous(), s) for (off, loc), s in zip(boxes, scales)]
    sources, handles = register_shards(shape, shards, granularity=g)
    want = torch.cat([torch_dequantize(box(q, off, loc).to(DEV), s.to(DEV), g, off[-2], off[-1], dst)
                      for (off, loc), s in zip(boxes, scales)], dim=-2)
    for c0, c1 in ((0, 200), (200, 520)):
        dest = torch.full((2, 300, c1 - c0), 7.0, dtype=dst, device=DEV)
        d = DirectWeightSyncDest()
        ts = TensorSlice((0, 0, c0), (0,), shape, (2, 300, c1 - c0), (2,))
        run(d.pull({"w": handles}, {"w": dest}, {"w": ts}))
        assert torch.equal(dest.view(torch.uint8), want[..., c0:c1].contiguous().view(torch.uint8))
        assert d._int8_dequant_plans and not d._dequant_plans
        d.close()
    cleanup(sources)


def verbatim_pull(handles, shape, g, ts=None, device=DEV):
    q = torch.full(shape, 0x55, dtype=torch.int8, device=device)
    s = torch.full(scale_shape(g, shape, 0, 0), -1.0, device=device)
    d = DirectWeightSyncDest()
    run(d.pull({"w": handles}, {"w": q}, None if ts is None else {"w": ts}, verbatim=True, **{KW[g]: {"w": s}}))
    d.close()
    return q, s


def quantising_pull(handles, shape, g, ts=None):
    q = torch.full(shape, 0x55, dtype=torch.int8, device=DEV)
    s = torch.full(scale_shape(g, shape, 0, 0), -1.0, device=DEV)
    d = DirectWeightSyncDest()
    run(d.pull({"w": handles}, {"w": q}, None if ts is None else {"w": ts}, **{KW[g]: {"w": s}}))
    d.close()
    return q, s


@pytest.mark.parametrize("g", GRANULARITIES)
def test_verbatim_int8_chain(g):
    """Source quantise -> verbatim pull into TP shards -> dequantise from the destination: every step keeps the
    source's int8 bytes and scales, so the final bf16 is the dequantised source staging."""
    shape = (512, 384)
    full = synth_f32(shape, 41).to(torch.bfloat16)
    if g == "tensor":  # one source group must hold every destination matrix
        src_boxes, tp = [((0, 0), shape)], ((0, 384),)
    elif g == "channel":
        src_boxes, tp = cols(shape, ()), ((0, 128), (128, 384))
    else:
        src_boxes, tp = rows(shape, (128, 384)), ((0, 256), (256, 384))
    sources, handles = register_boxes(full, src_boxes, quantize={"w": g}, quant_dtype=I8)
    want = torch.cat([torch_dequantize(*staging(src), g, off[0], off[1], torch.bfloat16)
                      for (src, *_), (off, _) in zip(sources, src_boxes)])
    for c0, c1 in tp:
        ts = TensorSlice((0, c0), (0,), shape, (512, c1 - c0), (2,))
        q, s = verbatim_pull(handles, (512, c1 - c0), g, ts)
        mid = DirectWeightSyncSource()
        h = mid.register({"w": q}, rank=0, tensor_slices={"w": ts}, **{KW[g]: {"w": s}})["w"]
        out = torch.zeros(512, c1 - c0, dtype=torch.bfloat16, device=DEV)
        d = DirectWeightSyncDest()
        run(d.pull({"w": [h]}, {"w": out}, {"w": ts}))
        assert torch.equal(out.view(torch.int16), want[:, c0:c1].contiguous().view(torch.int16))
        d.close()
        run(mid.cleanup())
    cleanup(sources)


@pytest.mark.parametrize("g", GRANULARITIES)
def test_unsharded_source_side_int8_equals_the_destination_side_pull(g):
    """Cross-check (b): with one group layout on both sides the two quantisers write the same bytes and scales."""
    shape = (3, 300, 260)
    full = synth_f32(shape, 51).to(torch.bfloat16)
    sources, handles = register_boxes(full, [((0, 0, 0), shape)], quantize={"w": g}, quant_dtype=I8)
    plain = DirectWeightSyncSource()
    ph = plain.register({"w": full.to(DEV)}, rank=0)["w"]
    dq, ds = quantising_pull([ph], shape, g)
    sq, ss = staging(sources[0][0])
    assert torch.equal(sq, dq) and torch.equal(ss.view(torch.int32), ds.reshape(ss.shape).view(torch.int32))
    vq, vs = verbatim_pull(handles, shape, g)
    assert torch.equal(vq, dq) and torch.equal(vs.view(torch.int32), ds.view(torch.int32))
    cleanup(sources + [(plain,)])


def test_mixed_pull_of_fp8_int8_quantising_and_plain_names():
    shape = (384, 256)
    fulls = {n: synth_f32(shape, 60 + i).to(torch.bfloat16) for i, n in enumerate(("f8", "i8", "i8v", "qz", "plain"))}
    sources, handles, by_name = [], {}, {}
    for n, qd in (("f8", E4M3), ("i8", torch.int8), ("i8v", torch.int8)):
        by_name[n], handles[n] = register_boxes(fulls[n], rows(shape, (128,)), name=n, quantize={n: "block"},
                                                quant_dtype=qd)
        sources += by_name[n]
    for n in ("qz", "plain"):
        src = DirectWeightSyncSource()
        handles[n] = [src.register({n: fulls[n].to(DEV)}, rank=0)[n]]
        sources.append((src,))
    dests = {"f8": torch.zeros(shape, dtype=torch.bfloat16, device=DEV),
             "i8": torch.zeros(shape, dtype=torch.float32, device=DEV),
             "i8v": torch.zeros(shape, dtype=torch.int8, device=DEV),
             "qz": torch.zeros(shape, dtype=torch.int8, device=DEV),
             "plain": torch.zeros(shape, dtype=torch.bfloat16, device=DEV)}
    bs = {"i8v": torch.full((3, 2), -1.0, device=DEV), "qz": torch.full((3, 2), -1.0, device=DEV)}
    d = DirectWeightSyncDest()
    for _ in range(2):  # built, then replayed
        run(d.pull(handles, dests, block_scales=bs, verbatim=True))
        from oracle.dequant_fp8_oracle import torch_dequantize as fp8_dequantize

        for n, dt in (("f8", torch.bfloat16), ("i8", torch.float32)):
            want = torch.cat([(fp8_dequantize if n == "f8" else torch_dequantize)(*staging(src, n), "block", r0, 0, dt)
                              for (src, *_), r0 in zip(by_name[n], (0, 128))])
            assert torch.equal(dests[n].view(torch.uint8), want.view(torch.uint8)), n
        vq = torch.cat([staging(src, "i8v")[0] for src, *_ in by_name["i8v"]])
        assert torch.equal(dests["i8v"], vq)
        tq, ts = torch_quantize(fulls["qz"].to(DEV), "block")
        assert torch.equal(dests["qz"], tq) and torch.equal(bs["qz"].view(torch.int32), ts.view(torch.int32))
        assert torch.equal(dests["plain"].cpu(), fulls["plain"])
    assert d._dequant_plans and d._int8_dequant_plans and d._int8_block_plans
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
            src = {"a": synth_f32((256, 384), 71).to(torch.bfloat16).to(DEV),
                   "b": synth_f32((2, 64, 300), 72).to(torch.float16).to(DEV)}
            await ts.put_state_dict(src, "policy_i8src", direct_rdma=True, quantize={"a": "block", "b": "tensor"},
                                    quant_dtype=torch.int8)
            dst = {"a": torch.zeros(256, 384, dtype=torch.int8, device=DEV),
                   "b": torch.zeros(2, 64, 300, dtype=torch.float32, device=DEV)}
            bs = {"a": torch.zeros(2, 3, device=DEV)}
            for _ in range(2):
                out = await ts.get_state_dict("policy_i8src", user_state_dict=dst, direct_rdma=True, block_scales=bs,
                                              verbatim=True)
                assert out is dst
                tq, tsc = torch_quantize(src["a"], "block")
                assert torch.equal(dst["a"], tq) and torch.equal(bs["a"].view(torch.int32), tsc.view(torch.int32))
                bq, bsc = torch_quantize(src["b"], "tensor")
                assert torch.equal(dst["b"], torch_dequantize(bq, bsc, "tensor", dst=torch.float32))
                src["a"].mul_(0.5)
                src["b"].mul_(3.0)
                await ts.put_state_dict(None, "policy_i8src", direct_rdma=True)
        finally:
            await ts.shutdown()
            dist.destroy_process_group()

    run(main())


def test_refusals_on_the_device():
    shape = (128, 256)
    full = synth_f32(shape, 81).to(torch.bfloat16)
    sources, handles = register_boxes(full, [((0, 0), shape)], quantize={"w": "channel"}, quant_dtype=I8)
    s = torch.zeros(128, 1, device=DEV)
    for kw in ({}, {"requantize": True}):
        with pytest.raises(TypeError, match="verbatim=True"):
            run(DirectWeightSyncDest().pull({"w": handles}, {"w": torch.zeros(shape, dtype=torch.int8, device=DEV)},
                                            channel_scales={"w": s}, **kw))
    for kw in ({}, {"requantize": True}, {"verbatim": True}):
        with pytest.raises(TypeError, match="int8 is not converted to fp8"):
            run(DirectWeightSyncDest().pull({"w": handles}, {"w": torch.zeros(shape, dtype=E4M3, device=DEV)},
                                            channel_scales={"w": s}, **kw))
    raw = torch.zeros(shape, dtype=torch.int8, device=DEV)  # not in a scale dict: the raw int8 bytes
    run(DirectWeightSyncDest().pull({"w": handles}, {"w": raw}))
    assert torch.equal(raw, staging(sources[0][0])[0])
    f8s, f8h = register_boxes(full, [((0, 0), shape)], quantize={"w": "channel"}, quant_dtype=E4M3)
    with pytest.raises(ValueError, match="mix scaled int8 and scaled fp8"):
        run(DirectWeightSyncDest().pull({"w": handles + f8h}, {"w": torch.zeros(shape, device=DEV)}))
    with pytest.raises(ValueError, match="int8 staging"):
        DirectWeightSyncSource().register({"w": full.to(DEV)}, rank=0, quantize={"w": "block"}, quant_dtype=torch.int8,
                                          scale_fmt="ue8m0")
    cleanup(sources + f8s)


@needs_two_gpus
@pytest.mark.parametrize("g", GRANULARITIES)
def test_fsdp_to_tp_over_peer_mappings(g):
    """Int8 staging quantised on cuda:0 and cuda:1 (FSDP(2) row shards), dequantised into TP(2) bf16 column shards
    and, for block, moved verbatim into TP(2) int8 column shards on both devices."""
    shape = (512, 768)
    full = synth_f32(shape, 91).to(torch.bfloat16)
    sources, handles = [], []
    for r, (off, loc) in enumerate(rows(shape, (256,))):
        s, h = register_boxes(full, [(off, loc)], device=f"cuda:{r}", quantize={"w": g}, quant_dtype=I8)
        sources += s
        handles += h
    want = torch.cat([torch_dequantize(*staging(src), g, r0, 0, torch.bfloat16).to(DEV)
                      for (src, *_), r0 in zip(sources, (0, 256))])
    for t in range(2):
        dev = f"cuda:{t}"
        c0, c1 = t * 384, (t + 1) * 384
        ts = TensorSlice((0, c0), (t,), shape, (512, 384), (2,))
        out = torch.zeros(512, 384, dtype=torch.bfloat16, device=dev)
        d = DirectWeightSyncDest()
        run(d.pull({"w": handles}, {"w": out}, {"w": ts}))
        assert torch.equal(out.cpu().view(torch.int16), want[:, c0:c1].cpu().contiguous().view(torch.int16))
        d.close()
        if g == "block":
            q, s = verbatim_pull(handles, (512, 384), g, ts, device=dev)
            want_q = torch.cat([staging(src)[0].to(DEV) for src, *_ in sources])[:, c0:c1]
            assert torch.equal(q.cpu(), want_q.cpu())
    cleanup(sources)


LLAMA3_8B = {"wq": (4096, 4096), "wk": (1024, 4096), "wv": (1024, 4096), "wo": (4096, 4096), "w1": (14336, 4096),
             "w2": (4096, 14336), "w3": (14336, 4096)}
COLUMN_PARALLEL = ("wq", "wk", "wv", "w1", "w3")


def fsdp_boxes(shape, n=8):
    step = shape[0] // n
    return [((r * step, 0), (step, shape[1])) for r in range(n)]


def tp_slice(name, shape, t, n=8):
    if name in COLUMN_PARALLEL:
        step = shape[0] // n
        return TensorSlice((t * step, 0), (t,), shape, (step, shape[1]), (n,))
    step = shape[1] // n
    return TensorSlice((0, t * step), (t,), shape, (shape[0], step), (n,))


@pytest.mark.parametrize("g", ("block", "channel"))
def test_llama3_8b_fsdp8_to_tp8_full_size(g):
    """Cross-check (a) at full size: FSDP(8) int8 staging pulled verbatim into TP(8) shards equals the
    destination-side int8 quantising pull of the same bf16 shards wherever each destination group is a source
    group (block everywhere, per channel on the column-parallel weights); every TP shard is also checked against
    the torch-CUDA rendering of its source shards."""
    names = LLAMA3_8B if g == "block" else {n: LLAMA3_8B[n] for n in COLUMN_PARALLEL}
    fulls = {n: (torch.randn(shape, device=DEV) * 0.02).to(torch.bfloat16) for n, shape in names.items()}
    sources, quant_h, plain_h = [], {n: [] for n in names}, {n: [] for n in names}
    for r in range(8):
        sd, sl = {}, {}
        for n, shape in names.items():
            off, loc = fsdp_boxes(shape)[r]
            sd[n] = box(fulls[n], off, loc).contiguous()
            sl[n] = TensorSlice(off, (r,), shape, loc, (8,))
        qs, ps = DirectWeightSyncSource(), DirectWeightSyncSource()
        qh = qs.register(sd, rank=r, tensor_slices=sl, quantize={n: g for n in names}, quant_dtype=torch.int8)
        ph = ps.register(sd, rank=r, tensor_slices=sl)
        for n in names:
            quant_h[n].append(qh[n])
            plain_h[n].append(ph[n])
        sources += [(qs,), (ps,)]
    staged = {n: torch.cat([src._quantized[n][0] for (src,) in sources[::2]]) for n in names}
    for t in range(8):
        dests, scales, ref_d, ref_s, tsl = {}, {}, {}, {}, {}
        for n, shape in names.items():
            tsl[n] = tp_slice(n, shape, t)
            loc = tuple(tsl[n].local_shape)
            dests[n], ref_d[n] = (torch.zeros(loc, dtype=torch.int8, device=DEV) for _ in range(2))
            scales[n], ref_s[n] = (torch.full(scale_shape(g, loc, 0, 0), -1.0, device=DEV) for _ in range(2))
        d, ref = DirectWeightSyncDest(), DirectWeightSyncDest()
        run(d.pull(quant_h, dests, tsl, verbatim=True, **{KW[g]: scales}))
        run(ref.pull(plain_h, ref_d, tsl, **{KW[g]: ref_s}))
        for n in names:
            assert torch.equal(dests[n], ref_d[n]), (n, t)
            assert torch.equal(scales[n].view(torch.int32), ref_s[n].view(torch.int32)), (n, t)
            (r0, c0), (nr, nc) = tsl[n].offsets, tsl[n].local_shape
            assert torch.equal(dests[n], staged[n][r0:r0 + nr, c0:c0 + nc]), (n, t)
        d.close()
        ref.close()
    for n in names:  # the staging itself against the torch-CUDA rendering, shard by shard
        for r, (src,) in enumerate(sources[::2]):
            (r0, c0), _ = fsdp_boxes(names[n])[r]
            tq, ts = torch_quantize(box(fulls[n], *fsdp_boxes(names[n])[r]), g, r0, c0)
            q, s = src._quantized[n][:2]
            assert torch.equal(q, tq) and torch.equal(s.view(torch.int32), ts.reshape(s.shape).view(torch.int32)), (n, r)
    cleanup(sources)

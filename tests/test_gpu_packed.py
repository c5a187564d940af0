"""Packed destinations on the GPU: HF-named trainer weights (FSDP shards simulated on cuda:0) pulled into vLLM's
fused qkv_proj / gate_up_proj and stacked MoE experts, checked bit for bit against the numpy oracle of the element
rule and against the unfused pull of the same bytes, through every route (byte copy, fused casts, quantising,
dequantising, requantising, verbatim), the plan cache and the public state-dict path."""

import numpy as np
import pytest
import torch

import workloads
from oracle import packed_oracle as po
from tests.helpers import (DEV, E4M3, as_np, masters, needs_two_gpus, nv_handles, pull, pull_args, region, run,
                           unfused_args, whole_handle)
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource, PackedPart, source_scale_shapes
from torchstore_b200.transport.types import TensorSlice

pytestmark = pytest.mark.gpu
LLAMA = workloads.LLAMA3_8B
QWEN = workloads.QWEN3_MOE


def fused(spec, shape, sources, dtype=None):
    """The element rule in torch, on the device: what a packed destination holds (zeros outside its parts)."""
    out = torch.zeros(shape, dtype=dtype or next(iter(sources.values())).dtype, device=DEV)
    for p in spec:
        box = out[p.dest_index]
        box.copy_(sources[p.source][tuple(slice(o, o + e) for o, e in zip(p.source_offsets, box.shape))])
    return out


# -- Llama-3 HF -> vLLM ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tp", [1, 2, 8])
def test_llama_hf_to_vllm_every_rank_bf16(tp):
    hf = workloads.hf_llama_layout(LLAMA, n_layers=2, scale=16)
    full = masters(hf, tp)
    handles = nv_handles(hf, 8, full)
    np_full = {k: as_np(v) for k, v in full.items()}
    for rank in range(tp):
        vl = workloads.vllm_tp_layout(hf, LLAMA, tp, rank)
        dests, slices, packed = pull_args(vl, tp, rank, lambda n, s: torch.full(s, -3, dtype=torch.int16, device=DEV)
                                          .view(torch.bfloat16))
        assert packed
        sync = pull(handles, dests, slices, packed=packed)
        for name, entry in vl.items():
            want = po.destination(entry, np_full, name, fill_value=-3, dtype=np.int16)
            assert np.array_equal(as_np(dests[name]), want), (rank, name)
        sync.close()


@pytest.mark.parametrize("staged", [False, True], ids=["fused_cast", "fp8_staging"])
def test_llama_into_fp8_destinations(staged):
    """bf16 handles cast to float8_e4m3fn during the pull, and transfer_dtype=float8_e4m3fn staging moved as bytes:
    either way every fused destination holds ``bf16.to(float8_e4m3fn)`` of its parts."""
    hf = workloads.hf_llama_layout(LLAMA, n_layers=1, scale=16)
    full = masters(hf, 21)
    if staged:
        srcs, handles = [], {}
        for r in range(8):
            sd, sl = {}, {}
            for name, (shape, _) in hf.items():
                off, loc = workloads.shard_box(shape, 8, r, ("S", 0))
                sd[name], sl[name] = region(full[name], off, loc).contiguous(), TensorSlice(off, (r,), shape, loc, (8,))
            src = DirectWeightSyncSource()
            for name, h in src.register(sd, rank=r, transfer_dtype=E4M3, tensor_slices=sl).items():
                handles.setdefault(name, []).append(h)
            srcs.append(src)
    else:
        handles = nv_handles(hf, 8, full)
    np_full = {k: as_np(v.to(E4M3)) for k, v in full.items()}
    for rank in (0, 1):
        vl = workloads.vllm_tp_layout(hf, LLAMA, 2, rank)
        dests, slices, packed = pull_args(vl, 2, rank, lambda n, s: torch.zeros(s, dtype=E4M3, device=DEV))
        sync = pull(handles, dests, slices, packed=packed)
        for name, entry in vl.items():
            assert np.array_equal(as_np(dests[name]), po.destination(entry, np_full, name)), (rank, name)
        sync.close()


def test_rename_only_part_equals_the_unpacked_pull():
    w = masters({"w": ((512, 384), None)}, 3)["w"]
    handles = nv_handles({"w": ((512, 384), None)}, 4, {"w": w})
    a = {"w": torch.zeros(512, 384, dtype=torch.bfloat16, device=DEV)}
    b = {"renamed": torch.zeros(512, 384, dtype=torch.bfloat16, device=DEV)}
    sa = pull(handles, a)
    sb = pull(handles, b, packed={"renamed": (PackedPart("w", (slice(None), slice(None)), (0, 0)),)})
    assert torch.equal(a["w"].view(torch.int16), b["renamed"].view(torch.int16))
    assert torch.equal(a["w"], w)
    assert sa.plan_info() == sb.plan_info()
    sa.close()
    sb.close()


@pytest.mark.parametrize("tp,rank", [(1, 0), (8, 3)])
def test_plan_info_equals_the_unfused_pull(tp, rank):
    """The packed pull compiles to the device work of the unfused pull of the same bytes: same rects, vector rects,
    tiles, copy/link split and bytes; and the unfused destinations hold exactly the parts' boxes."""
    hf = workloads.hf_llama_layout(LLAMA, n_layers=2, scale=8)
    full = masters(hf, 5)
    handles = nv_handles(hf, 8, full)
    vl = workloads.vllm_tp_layout(hf, LLAMA, tp, rank)
    mk = lambda n, s: torch.zeros(s, dtype=torch.bfloat16, device=DEV)  # noqa: E731
    dests, slices, packed = pull_args(vl, tp, rank, mk)
    udests, uslices, where = unfused_args(vl, hf, tp, rank, mk)
    sp, su = pull(handles, dests, slices, packed=packed), pull(handles, udests, uslices)
    assert sp.plan_info() == su.plan_info()
    for name, parts in where.items():
        for p, uname in parts:
            assert torch.equal(dests[name][p.dest_index], udests[uname]), (name, uname)
    sp.close()
    su.close()


# -- quantising into fused destinations ------------------------------------------------------------------------------
QUANT_CASES = [(dt, g, fmt) for dt in (E4M3, torch.int8) for g in ("block", "channel", "tensor")
               for fmt in ((None, "ue8m0") if dt == E4M3 else (None,))]


@pytest.mark.parametrize("dtype,g,fmt", QUANT_CASES, ids=[f"{'fp8' if d == E4M3 else 'int8'}-{g}-{f}" for d, g, f in QUANT_CASES])
def test_quantising_into_fused_destinations(dtype, g, fmt):
    """qkv_proj / gate_up_proj quantised during the pull equal an unpacked pull from one handle over the fused
    high-precision tensor: the groups span the parts (per tensor: one amax over q, k and v together)."""
    hf = workloads.hf_llama_layout(LLAMA, n_layers=1, scale=16, with_embeddings=False)
    full = masters(hf, 31)
    handles = nv_handles(hf, 4, full)
    vl = workloads.vllm_tp_layout(hf, LLAMA, 2, 1)
    for name, (shape, parts, _) in vl.items():
        if parts is None:
            continue
        q = torch.zeros(shape, dtype=dtype, device=DEV)
        s = torch.full(source_scale_shapes(g, shape, 0, 0)[0], -1.0, device=DEV)
        sync = pull(handles, {name: q}, packed={name: parts}, **{f"{g}_scales": {name: s}}, scale_fmt=fmt)
        ref_q, ref_s = torch.zeros_like(q), torch.full_like(s, -2.0)
        ref = pull({name: whole_handle(fused(parts, shape, full))}, {name: ref_q}, **{f"{g}_scales": {name: ref_s}},
                   scale_fmt=fmt)
        assert torch.equal(q.view(torch.uint8), ref_q.view(torch.uint8)), name
        assert torch.equal(s.view(torch.int32), ref_s.view(torch.int32)), name
        sync.close()
        ref.close()


# -- scaled sources: dequantising, requantising, verbatim ---------------------------------------------------------
SCALED = {"q": (512, 256), "k": (256, 256), "v": (256, 256), "gate": (512, 256), "up": (512, 256)}
SCALED_PACKED = {
    "qkv": ((1024, 256), (PackedPart("q", (slice(0, 512), slice(0, 256)), (0, 0)),
                          PackedPart("k", (slice(512, 768), slice(0, 256)), (0, 0)),
                          PackedPart("v", (slice(768, 1024), slice(0, 256)), (0, 0)))),
    # TP2 rank 1's halves of gate and up
    "gate_up": ((512, 256), (PackedPart("gate", (slice(0, 256), slice(0, 256)), (256, 0)),
                             PackedPart("up", (slice(256, 512), slice(0, 256)), (256, 0)))),
}


def scaled_sources(g, qdtype, seed):
    """q/k/v/gate/up quantised on the source (register(quantize=...)) in FSDP(2) row shards -> (handles, sources,
    global staging, global scale (block and channel: the shards' scales stacked))."""
    layout = {n: (s, None) for n, s in SCALED.items()}
    full = masters(layout, seed)
    srcs, handles, gq, gs = [], {}, {}, {}
    for r in range(2):
        sd, sl = {}, {}
        for name, (shape, _) in layout.items():
            off, loc = workloads.shard_box(shape, 2, r, ("S", 0))
            sd[name], sl[name] = region(full[name], off, loc).contiguous(), TensorSlice(off, (r,), shape, loc, (2,))
        src = DirectWeightSyncSource()
        for name, h in src.register(sd, rank=r, tensor_slices=sl, quantize={n: g for n in sd},
                                    quant_dtype=qdtype).items():
            handles.setdefault(name, []).append(h)
        srcs.append(src)
    for name in layout:
        gq[name] = torch.cat([s._quantized[name][0] for s in srcs])
        if g != "tensor":
            gs[name] = torch.cat([s._quantized[name][1] for s in srcs])
    return handles, srcs, gq, gs


def unfused_dequant(handles, name, shape, parts, dtype):
    """Each part pulled on its own (unpacked) into a destination of its box, placed where the part goes."""
    out = torch.zeros(shape, dtype=dtype, device=DEV)
    for p in parts:
        box = out[p.dest_index]
        d = torch.zeros(box.shape, dtype=dtype, device=DEV)
        gshape = handles[p.source][0].tensor_slice.global_shape
        sync = pull(handles, {p.source: d}, {p.source: TensorSlice(p.source_offsets, (0,), gshape, tuple(box.shape), (1,))})
        box.copy_(d)
        sync.close()
    return out


@pytest.mark.parametrize("qdtype", [E4M3, torch.int8], ids=["fp8", "int8"])
@pytest.mark.parametrize("g", ["block", "channel", "tensor"])
def test_dequantising_into_fused_destinations(qdtype, g):
    handles, srcs, _, _ = scaled_sources(g, qdtype, 41)
    for dtype in (torch.bfloat16, torch.float32):
        for name, (shape, parts) in SCALED_PACKED.items():
            d = torch.full(shape, 7.0, dtype=dtype, device=DEV)
            sync = pull(handles, {name: d}, packed={name: parts})
            assert sync._int8_dequant_plans if qdtype == torch.int8 else sync._dequant_plans
            assert torch.equal(d, unfused_dequant(handles, name, shape, parts, dtype)), (name, dtype)
            sync.close()


@pytest.mark.parametrize("g", ["block", "channel", "tensor"])
def test_requantising_into_fused_destinations(g):
    """A requantising packed pull equals a dequantising packed pull into float32 followed by a quantising pull
    from it."""
    handles, srcs, _, _ = scaled_sources(g, E4M3, 42)
    for dg in ("block", "channel", "tensor"):
        for name, (shape, parts) in SCALED_PACKED.items():
            q = torch.zeros(shape, dtype=E4M3, device=DEV)
            s = torch.full(source_scale_shapes(dg, shape, 0, 0)[0], -1.0, device=DEV)
            sync = pull(handles, {name: q}, packed={name: parts}, requantize=True, **{f"{dg}_scales": {name: s}})
            f32 = torch.zeros(shape, dtype=torch.float32, device=DEV)
            pull(handles, {name: f32}, packed={name: parts}).close()
            ref_q, ref_s = torch.zeros_like(q), torch.full_like(s, -2.0)
            pull({name: whole_handle(f32)}, {name: ref_q}, **{f"{dg}_scales": {name: ref_s}}).close()
            assert torch.equal(q.view(torch.uint8), ref_q.view(torch.uint8)), (name, dg)
            assert torch.equal(s.view(torch.int32), ref_s.view(torch.int32)), (name, dg)
            sync.close()


@pytest.mark.parametrize("qdtype", [E4M3, torch.int8], ids=["fp8", "int8"])
@pytest.mark.parametrize("g", ["block", "channel"])
def test_verbatim_into_fused_destinations(qdtype, g):
    """The source's bytes and the scales of the source groups holding each destination group, as they are."""
    handles, srcs, gq, gs = scaled_sources(g, qdtype, 43)
    step = 128 if g == "block" else 1
    for name, (shape, parts) in SCALED_PACKED.items():
        q = torch.zeros(shape, dtype=qdtype, device=DEV)
        s = torch.full(source_scale_shapes(g, shape, 0, 0)[0], -1.0, device=DEV)
        sync = pull(handles, {name: q}, packed={name: parts}, verbatim=True, **{f"{g}_scales": {name: s}})
        assert not any(sync._fp8_plans)
        assert torch.equal(q.view(torch.uint8), fused(parts, shape, gq).view(torch.uint8)), name
        scale_parts = [PackedPart(p.source, (slice(p.dest_index[0].start // step, p.dest_index[0].stop // step),
                                             slice(0, gs[p.source].shape[1])), (p.source_offsets[0] // step, 0))
                       for p in parts]
        assert torch.equal(s.view(torch.int32), fused(scale_parts, tuple(s.shape), gs).view(torch.int32)), name
        sync.close()


# -- MoE stacks -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["tp2", "ep2"])
def test_moe_experts_into_stacks(mode):
    hf = workloads.qwen3_moe_layout(QWEN, n_layers=1, scale=8, n_experts=4)
    full = masters(hf, 51)
    handles = nv_handles(hf, 2, full)
    np_full = {k: as_np(v) for k, v in full.items()}
    for rank in range(2):
        vl = workloads.vllm_tp_layout(hf, QWEN, 2, rank, ep=mode == "ep2")
        dests, slices, packed = pull_args(vl, 2, rank, lambda n, s: torch.full(s, -3, dtype=torch.int16, device=DEV)
                                          .view(torch.bfloat16))
        assert dests["model.layers.0.mlp.experts.w13_weight"].shape[0] == (2 if mode == "ep2" else 4)
        sync = pull(handles, dests, slices, packed=packed)
        for name, entry in vl.items():
            want = po.destination(entry, np_full, name, fill_value=-3, dtype=np.int16)
            assert np.array_equal(as_np(dests[name]), want), (rank, name)
        sync.close()


def test_moe_per_tensor_scales_per_expert():
    """w13_weight / w2_weight with one scale per expert ([E]) quantise each expert's fused matrix on its own."""
    hf = workloads.qwen3_moe_layout(QWEN, n_layers=1, scale=8, n_experts=4, with_embeddings=False)
    full = masters(hf, 52)
    handles = nv_handles(hf, 2, full)
    vl = workloads.vllm_tp_layout(hf, QWEN, 2, 1)
    for name in ("model.layers.0.mlp.experts.w13_weight", "model.layers.0.mlp.experts.w2_weight"):
        shape, parts, _ = vl[name]
        q, s = torch.zeros(shape, dtype=E4M3, device=DEV), torch.full((shape[0],), -1.0, device=DEV)
        sync = pull(handles, {name: q}, packed={name: parts}, tensor_scales={name: s})
        ref_q, ref_s = torch.zeros_like(q), torch.full_like(s, -2.0)
        pull({name: whole_handle(fused(parts, shape, full))}, {name: ref_q}, tensor_scales={name: ref_s}).close()
        assert torch.equal(q.view(torch.uint8), ref_q.view(torch.uint8)), name
        assert torch.equal(s.view(torch.int32), ref_s.view(torch.int32)), name
        sync.close()


def test_moe_verbatim_block_straddling_two_parts_is_refused():
    """Qwen3-30B-A3B's w13 at TP8 holds 96-row gate and up halves: block row 0 of each expert straddles both."""
    full = masters({"gate": ((768, 256), None), "up": ((768, 256), None)}, 53)
    src = DirectWeightSyncSource()
    handles = {n: [h] for n, h in src.register(full, rank=0, quantize={"gate": "block", "up": "block"}).items()}
    parts = (PackedPart("gate", (0, slice(0, 96), slice(0, 256)), (96, 0)),
             PackedPart("up", (0, slice(96, 192), slice(0, 256)), (96, 0)))
    q = torch.zeros(1, 192, 256, dtype=E4M3, device=DEV)
    s = torch.zeros(source_scale_shapes("block", (1, 192, 256), 0, 0)[0], device=DEV)
    sync = DirectWeightSyncDest()
    with pytest.raises(ValueError, match=r"verbatim pull of 'w13' \(block_scales\): destination block \(0, 0, 0\)"):
        run(sync.pull(handles, {"w13": q}, packed={"w13": parts}, block_scales={"w13": s}, verbatim=True))
    assert sync._plan is None
    # requantize=True pulls it into the destination's blocks
    run(sync.pull(handles, {"w13": q}, packed={"w13": parts}, block_scales={"w13": s}, requantize=True))
    assert (s > 0).all()
    sync.close()


# -- plan cache -----------------------------------------------------------------------------------------------------
def test_plan_cache(monkeypatch):
    builds = []
    orig = DirectWeightSyncDest._build_plan
    monkeypatch.setattr(DirectWeightSyncDest, "_build_plan", lambda self, *a, **k: builds.append(1) or orig(self, *a, **k))
    full = masters({"a": ((256, 128), None), "b": ((256, 128), None)}, 61)
    handles = nv_handles({"a": ((256, 128), None), "b": ((256, 128), None)}, 2, full)
    spec = (PackedPart("a", (slice(0, 256), slice(0, 128)), (0, 0)), PackedPart("b", (slice(256, 512), slice(0, 128)), (0, 0)))
    dests = {"ab": torch.zeros(512, 128, dtype=torch.bfloat16, device=DEV)}
    packed = {"ab": spec}
    sync = DirectWeightSyncDest()
    for _ in range(3):
        run(sync.pull(handles, dests, packed=packed))
    assert len(builds) == 1
    assert torch.equal(dests["ab"], torch.cat([full["a"], full["b"]]))
    run(sync.pull(handles, dests, packed={"ab": tuple(spec)}))  # a fresh dict with equal content keeps the plan
    run(sync.pull(handles, dests, packed={"ab": spec[:1] + (PackedPart("b", (slice(256, 512), slice(0, 128)), (0, 0)),)}))
    assert len(builds) == 1
    packed["ab"] = (PackedPart("b", (slice(0, 256), slice(0, 128)), (0, 0)), PackedPart("a", (slice(256, 512), slice(0, 128)), (0, 0)))
    run(sync.pull(handles, dests, packed=packed))  # the same dict, edited: rebuilt
    assert len(builds) == 2
    assert torch.equal(dests["ab"], torch.cat([full["b"], full["a"]]))
    run(sync.pull(handles, dests, packed=packed))
    assert len(builds) == 2
    sync.close()


# -- the public path --------------------------------------------------------------------------------------------------
def test_get_state_dict_with_packed():
    import torch.distributed as dist
    from torch.testing._internal.distributed.fake_pg import FakeStore

    import torchstore_b200 as ts

    hf = workloads.hf_llama_layout(LLAMA, n_layers=1, scale=16, with_embeddings=False)
    full = masters(hf, 71)
    vl = workloads.vllm_tp_layout(hf, LLAMA, 1, 0)
    packed = {n: parts for n, (_, parts, _) in vl.items() if parts}

    async def main():
        dist.init_process_group("fake", store=FakeStore(), rank=0, world_size=1)
        await ts.initialize()
        try:
            await ts.put_state_dict(full, "policy_packed", direct_rdma=True)
            dst = {n: torch.zeros(vl[n][0], dtype=torch.bfloat16, device=DEV) for n in packed}
            for _ in range(2):
                out = await ts.get_state_dict("policy_packed", user_state_dict=dst, direct_rdma=True, packed=packed)
                assert out is dst
                for n, parts in packed.items():
                    assert torch.equal(dst[n], fused(parts, vl[n][0], full)), n
                for t in full.values():
                    t.mul_(2)
            with pytest.raises(NotImplementedError, match="packed"):
                await ts.get_state_dict("policy_packed", user_state_dict=dst, packed=packed)
        finally:
            await ts.shutdown()
            dist.destroy_process_group()

    run(main())


@needs_two_gpus
def test_parts_read_over_peer_mappings():
    """Parts whose handles live on cuda:1 are read over NVLink by cuda:0's copy plan (the link queue)."""
    hf = workloads.hf_llama_layout(LLAMA, n_layers=1, scale=8, with_embeddings=False)
    full = masters(hf, 81, device="cuda:1")
    handles = nv_handles(hf, 2, full)
    vl = workloads.vllm_tp_layout(hf, LLAMA, 2, 0)
    dests, slices, packed = pull_args(vl, 2, 0, lambda n, s: torch.zeros(s, dtype=torch.bfloat16, device=DEV))
    sync = pull(handles, dests, slices, packed=packed)
    info = sync.plan_info()[0]
    assert info["remote_src_bytes"] > 0 and info["num_link_tiles"] > 0
    for n, parts in packed.items():
        want = fused(parts, vl[n][0], {k: v.to(DEV) for k, v in full.items()})
        assert torch.equal(dests[n], want), n
    sync.close()

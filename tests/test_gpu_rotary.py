"""Rotary packed parts on the GPU: a torchtitan trainer's interleaved wq / wk (FSDP shards simulated on cuda:0) pulled
into vLLM's half-split qkv_proj through every route.  Byte copies and casts are checked bit for bit against
rotary_oracle (alone, or composed with packed_oracle); the grouped and scaled routes against the HF-named packed pull
of the same weights with their heads permuted by torch (``view / transpose / reshape``), whose routes the packed
suites check against their own oracles."""

import numpy as np
import pytest
import torch

import workloads
from oracle import packed_oracle as po
from oracle import rotary_oracle as ro
from tests.helpers import (DEV, E4M3, as_np, masters, needs_two_gpus, nv_handles, pull, pull_args, region, run,
                           whole_handle)
from torchstore_b200.direct_weight_sync import (DirectWeightSyncDest, DirectWeightSyncSource, PackedPart,
                                                RDMAWeightHandle, source_scale_shapes)
from torchstore_b200.transport.types import TensorSlice

pytestmark = pytest.mark.gpu
LLAMA = workloads.LLAMA3_8B


def half_split(t, hd):
    """The torch conversion of torchtitan's (and HF's) checkpoint scripts, per head along dim -2."""
    rows, cols = t.shape[-2:]
    return t.view(rows // hd, hd // 2, 2, cols).transpose(1, 2).reshape(rows, cols)


def titan(layout_scale=16, n_layers=2, with_embeddings=True):
    return workloads.llama_layout(LLAMA, n_layers=n_layers, scale=layout_scale, with_embeddings=with_embeddings)


def i16(shape):
    return torch.full(shape, -3, dtype=torch.int16, device=DEV).view(torch.bfloat16)


# -- bf16 and casts, against rotary_oracle ----------------------------------------------------------------------------
@pytest.mark.parametrize("tp,n", [(1, 8), (2, 8), (8, 8), (2, 3), (8, 3)])
def test_llama_torchtitan_to_vllm_every_rank_bf16(tp, n):
    """Scaled-down Llama-3 (dim 256, hd 8), torchtitan FSDP(n) -> vLLM TP(tp), every rank and every parameter.
    FSDP(3)'s uneven shards cut through heads."""
    layout = titan()
    full = masters(layout, tp * 10 + n)
    handles = nv_handles(layout, n, full)
    np_full = {k: as_np(v) for k, v in full.items()}
    for rank in range(tp):
        vl = workloads.vllm_tp_layout(layout, LLAMA, tp, rank, source="torchtitan")
        dests, _, packed = pull_args(vl, tp, rank, lambda _, s: i16(s))
        sync = pull(handles, dests, packed=packed)
        for name, entry in vl.items():
            want = ro.destination(entry, np_full, name, fill_value=-3, dtype=np.int16)
            assert np.array_equal(as_np(dests[name]), want), (rank, name)
        sync.close()


@pytest.mark.parametrize("staged", [False, True], ids=["fused_cast", "fp8_staging"])
def test_llama_into_fp8_destinations(staged):
    """bf16 handles cast to float8_e4m3fn in the pull, or transfer_dtype=float8_e4m3fn staging moved as bytes: the
    fused parameters hold rotary_oracle composed with packed_oracle over ``bf16.to(float8_e4m3fn)``."""
    layout = titan(n_layers=1)
    full = masters(layout, 21)
    if staged:
        srcs, handles = [], {}
        for r in range(8):
            sd, sl = {}, {}
            for name, (shape, _) in layout.items():
                off, loc = workloads.shard_box(shape, 8, r, ("S", 0))
                sd[name], sl[name] = region(full[name], off, loc).contiguous(), TensorSlice(off, (r,), shape, loc, (8,))
            src = DirectWeightSyncSource()
            for name, h in src.register(sd, rank=r, transfer_dtype=E4M3, tensor_slices=sl).items():
                handles.setdefault(name, []).append(h)
            srcs.append(src)
    else:
        handles = nv_handles(layout, 8, full)
    np_full = {k: as_np(v.to(E4M3)) for k, v in full.items()}
    for rank in (0, 1):
        vl = workloads.vllm_tp_layout(layout, LLAMA, 2, rank, source="torchtitan")
        dests, _, packed = pull_args(vl, 2, rank, lambda _, s: torch.zeros(s, dtype=E4M3, device=DEV))
        sync = pull(handles, dests, packed=packed)
        for name, (shape, parts, _) in vl.items():
            plain_parts, plain_sources = ro.plain(parts, np_full)
            want = po.fill(np.zeros(shape, dtype=np.uint8), plain_parts, plain_sources)
            assert np.array_equal(as_np(dests[name]), want), (rank, name)
        sync.close()


# -- a Qwen3-MoE-shaped attention (hd 128) through the grouped and scaled routes --------------------------------------
HD = 128
ATTN = {"wq": (32 * HD, 256), "wk": (4 * HD, 256), "wv": (4 * HD, 256)}
# TP2 rank 1: query heads 16..31, kv heads 2..3
ROTARY = (PackedPart("wq", (slice(0, 2048), slice(0, 256)), (2048, 0), rotary_head_dim=HD),
          PackedPart("wk", (slice(2048, 2304), slice(0, 256)), (256, 0), rotary_head_dim=HD),
          PackedPart("wv", (slice(2304, 2560), slice(0, 256)), (256, 0)))
PLAIN = tuple(PackedPart(p.source + "_hf", p.dest_index, p.source_offsets) for p in ROTARY)
SHAPE = (2560, 256)


def attention(seed):
    """torchtitan-ordered wq / wk / wv and their HF-ordered twins (``*_hf``: heads permuted by torch)."""
    full = masters({n: (s, None) for n, s in ATTN.items()}, seed)
    full.update({f"{n}_hf": half_split(full[n], HD) if n != "wv" else full[n] for n in ATTN})
    return full


def rotary_fill(full, dtype=torch.bfloat16):
    """The rotary element rule on the device, in torch."""
    out = torch.zeros(SHAPE, dtype=dtype, device=DEV)
    for p in PLAIN:
        box = out[p.dest_index]
        box.copy_(full[p.source][p.source_offsets[0]:p.source_offsets[0] + box.shape[0]])
    return out


QUANT_CASES = [(dt, g, fmt) for dt in (E4M3, torch.int8) for g in ("block", "channel", "tensor")
               for fmt in ((None, "ue8m0") if dt == E4M3 else (None,))]


@pytest.mark.parametrize("dtype,g,fmt", QUANT_CASES, ids=[f"{'fp8' if d == E4M3 else 'int8'}-{g}-{f}" for d, g, f in QUANT_CASES])
def test_quantising_into_rotary_qkv(dtype, g, fmt):
    """Quantised during the pull from interleaved bf16 handles: equal to the pull of one handle over the fused
    half-split tensor (the destination's groups span the parts)."""
    full = attention(31)
    handles = nv_handles({n: (s, None) for n, s in ATTN.items()}, 2, full)
    q = torch.zeros(SHAPE, dtype=dtype, device=DEV)
    s = torch.full(source_scale_shapes(g, SHAPE, 0, 0)[0], -1.0, device=DEV)
    sync = pull(handles, {"qkv": q}, packed={"qkv": ROTARY}, **{f"{g}_scales": {"qkv": s}}, scale_fmt=fmt)
    ref_q, ref_s = torch.zeros_like(q), torch.full_like(s, -2.0)
    pull({"qkv": whole_handle(rotary_fill(full))}, {"qkv": ref_q}, **{f"{g}_scales": {"qkv": ref_s}},
         scale_fmt=fmt).close()
    assert torch.equal(q.view(torch.uint8), ref_q.view(torch.uint8))
    assert torch.equal(s.view(torch.int32), ref_s.view(torch.int32))
    sync.close()


def scaled_attention(g, qdtype, seed, n=2):
    """wq / wk / wv and their HF twins quantised on the source (register(quantize=...)) in FSDP(n) row shards."""
    full = attention(seed)
    srcs, handles = [], {}
    for r in range(n):
        sd, sl = {}, {}
        for name, t in full.items():
            off, loc = workloads.shard_box(tuple(t.shape), n, r, ("S", 0))
            sd[name], sl[name] = region(t, off, loc).contiguous(), TensorSlice(off, (r,), tuple(t.shape), loc, (n,))
        src = DirectWeightSyncSource()
        for name, h in src.register(sd, rank=r, tensor_slices=sl, quantize={k: g for k in sd}, quant_dtype=qdtype).items():
            handles.setdefault(name, []).append(h)
        srcs.append(src)
    return handles, srcs


@pytest.mark.parametrize("qdtype", [E4M3, torch.int8], ids=["fp8", "int8"])
@pytest.mark.parametrize("g", ["block", "channel", "tensor"])
def test_dequantising_rotary_parts(qdtype, g):
    """Scaled handles of interleaved weights dequantised into the half-split qkv_proj equal the HF-named packed pull
    from the scaled handles of the torch-permuted weights (a head's rows share their blocks, rows keep their channel
    scales, a shard keeps its tensor scale)."""
    handles, srcs = scaled_attention(g, qdtype, 41)
    for dtype in (torch.bfloat16, torch.float32):
        a, b = torch.full(SHAPE, 7.0, dtype=dtype, device=DEV), torch.full(SHAPE, 5.0, dtype=dtype, device=DEV)
        sync = pull(handles, {"qkv": a}, packed={"qkv": ROTARY})
        assert sync._int8_dequant_plans if qdtype == torch.int8 else sync._dequant_plans
        pull(handles, {"qkv": b}, packed={"qkv": PLAIN}).close()
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), dtype
        sync.close()


@pytest.mark.parametrize("g", ["block", "channel", "tensor"])
def test_requantising_rotary_parts(g):
    handles, srcs = scaled_attention(g, E4M3, 42)
    for dg in ("block", "channel", "tensor"):
        outs = []
        for spec in (ROTARY, PLAIN):
            q = torch.zeros(SHAPE, dtype=E4M3, device=DEV)
            s = torch.full(source_scale_shapes(dg, SHAPE, 0, 0)[0], -1.0, device=DEV)
            pull(handles, {"qkv": q}, packed={"qkv": spec}, requantize=True, **{f"{dg}_scales": {"qkv": s}}).close()
            outs.append((q.view(torch.uint8), s.view(torch.int32)))
        assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1]), dg


@pytest.mark.parametrize("qdtype", [E4M3, torch.int8], ids=["fp8", "int8"])
@pytest.mark.parametrize("g", ["block", "channel"])
def test_verbatim_rotary_parts(qdtype, g):
    """Bytes and the scales of the source groups holding each destination group, as they are: block scales stay (hd
    128 divides the block), channel scales move with their rows."""
    handles, srcs = scaled_attention(g, qdtype, 43)
    outs = []
    for spec in (ROTARY, PLAIN):
        q = torch.zeros(SHAPE, dtype=qdtype, device=DEV)
        s = torch.full(source_scale_shapes(g, SHAPE, 0, 0)[0], -1.0, device=DEV)
        sync = pull(handles, {"qkv": q}, packed={"qkv": spec}, verbatim=True, **{f"{g}_scales": {"qkv": s}})
        assert not any(sync._fp8_plans)
        sync.close()
        outs.append((q.view(torch.uint8), s.view(torch.int32)))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


@pytest.mark.parametrize("g", ["block", "channel", "tensor"])
def test_fsdp3_shards_cut_heads_on_scaled_routes(g):
    """FSDP(3) shards of wq end inside heads: dequantising and requantising still equal the HF-named pull (the
    permuted twins are cut at the same rows, so they are compared through bf16 handles quantised on the destination,
    and through dequantising into float32 against the fused rule applied to each shard's dequantised values)."""
    full = attention(44)
    handles = nv_handles({n: (tuple(t.shape), None) for n, t in full.items()}, 3, full)
    q = torch.zeros(SHAPE, dtype=E4M3, device=DEV)
    s = torch.full(source_scale_shapes(g, SHAPE, 0, 0)[0], -1.0, device=DEV)
    pull(handles, {"qkv": q}, packed={"qkv": ROTARY}, **{f"{g}_scales": {"qkv": s}}).close()
    ref_q, ref_s = torch.zeros_like(q), torch.full_like(s, -2.0)
    pull(handles, {"qkv": ref_q}, packed={"qkv": PLAIN}, **{f"{g}_scales": {"qkv": ref_s}}).close()
    assert torch.equal(q.view(torch.uint8), ref_q.view(torch.uint8)) and torch.equal(s, ref_s)
    # scaled FSDP(3) handles: the rotary dequantising pull equals each shard dequantised by torch, then reordered
    shandles, srcs = scaled_attention(g, E4M3, 45, n=3)
    out = torch.zeros(SHAPE, dtype=torch.float32, device=DEV)
    pull(shandles, {"qkv": out}, packed={"qkv": ROTARY}).close()
    deq = {}
    for name in ATTN:
        rows = []
        for h in shandles[name]:
            buf = h.rdma_buffer
            w = torch.zeros(buf.shape, dtype=torch.float32, device=DEV)
            pull({name: [RDMAWeightHandle(buf, TensorSlice((0, 0), (0,), buf.shape, buf.shape, (1,)), 0)]},
                 {name: w}).close()
            rows.append(w)
        deq[name] = torch.cat(rows)
    want = ro.fill(np.zeros(SHAPE, dtype=np.float32), ROTARY, {k: v.cpu().numpy() for k, v in deq.items()})
    assert np.array_equal(out.cpu().numpy().view(np.int32), want.view(np.int32))


# -- plan cache, full size, public path, peers ------------------------------------------------------------------------
def test_plan_rebuilds_when_the_head_dim_changes(monkeypatch):
    builds = []
    orig = DirectWeightSyncDest._build_plan
    monkeypatch.setattr(DirectWeightSyncDest, "_build_plan", lambda self, *a, **k: builds.append(1) or orig(self, *a, **k))
    full = attention(61)
    handles = nv_handles({n: (s, None) for n, s in ATTN.items()}, 2, full)
    d = {"qkv": torch.zeros(SHAPE, dtype=torch.bfloat16, device=DEV)}
    sync = DirectWeightSyncDest()
    for hd, want in ((HD, rotary_fill(full)), (None, None), (HD, rotary_fill(full))):
        spec = tuple(PackedPart(p.source, p.dest_index, p.source_offsets, hd if p.rotary_head_dim else None) for p in ROTARY)
        run(sync.pull(handles, d, packed={"qkv": spec}))
        run(sync.pull(handles, d, packed={"qkv": spec}))
        if want is None:  # rows in source order
            want = torch.cat([full["wq"][2048:], full["wk"][256:], full["wv"][256:]])
        assert torch.equal(d["qkv"], want), hd
    assert len(builds) == 3
    sync.close()


def test_full_size_llama3_8b_one_rank():
    """Full-size Llama-3-8B layer 0 (hd 128), torchtitan FSDP(8) -> vLLM TP8 rank 3, bf16, against rotary_oracle."""
    layout = workloads.llama_layout(LLAMA, n_layers=1, with_embeddings=False)
    full = masters(layout, 91)
    handles = nv_handles(layout, 8, full)
    vl = workloads.vllm_tp_layout(layout, LLAMA, 8, 3, source="torchtitan")
    dests, _, packed = pull_args(vl, 8, 3, lambda _, s: i16(s))
    sync = pull(handles, dests, packed=packed)
    np_full = {k: as_np(v) for k, v in full.items()}
    for name, entry in vl.items():
        assert np.array_equal(as_np(dests[name]), ro.destination(entry, np_full, name, fill_value=-3, dtype=np.int16)), name
    sync.close()


@needs_two_gpus
def test_rotary_parts_read_over_peer_mappings():
    layout = titan(layout_scale=8, n_layers=1, with_embeddings=False)
    full = masters(layout, 81, device="cuda:1")
    handles = nv_handles(layout, 2, full)
    vl = workloads.vllm_tp_layout(layout, LLAMA, 2, 0, source="torchtitan")
    dests, _, packed = pull_args(vl, 2, 0, lambda _, s: i16(s))
    sync = pull(handles, dests, packed=packed)
    assert sync.plan_info()[0]["remote_src_bytes"] > 0
    np_full = {k: as_np(v) for k, v in full.items()}
    for name, entry in vl.items():
        assert np.array_equal(as_np(dests[name]), ro.destination(entry, np_full, name, fill_value=-3, dtype=np.int16)), name
    sync.close()


@pytest.mark.parametrize("tp,rank", [(1, 0), (8, 3)])
def test_plan_info_equals_the_hf_named_packed_pull(tp, rank):
    """The torchtitan rotary pull moves the same bytes with the same copy/link split as the HF-named packed pull of
    the same layout; both rect counts are reported."""
    layout = titan(layout_scale=8, n_layers=2)
    full = masters(layout, 5)
    hf_full = {workloads.hf_name(k): v for k, v in full.items()}  # the bytes, not the values, matter here
    handles = nv_handles(layout, 8, full)
    hf = workloads.hf_llama_layout(LLAMA, n_layers=2, scale=8)
    hf_handles = nv_handles(hf, 8, hf_full)
    vt = workloads.vllm_tp_layout(layout, LLAMA, tp, rank, source="torchtitan")
    vh = workloads.vllm_tp_layout(hf, LLAMA, tp, rank)
    dt, _, pt = pull_args(vt, tp, rank, lambda _, s: torch.zeros(s, dtype=torch.bfloat16, device=DEV))
    dh, sh, ph = pull_args(vh, tp, rank, lambda _, s: torch.zeros(s, dtype=torch.bfloat16, device=DEV))
    st, sh_ = pull(handles, dt, packed=pt), pull(hf_handles, dh, sh, packed=ph)
    it, ih = st.plan_info()[0], sh_.plan_info()[0]
    print({"torchtitan_rotary_rects": it.get("num_rects"), "hf_packed_rects": ih.get("num_rects")})
    for key in it:
        if "byte" in key or "link" in key:
            assert it[key] == ih[key], key
    st.close()
    sh_.close()

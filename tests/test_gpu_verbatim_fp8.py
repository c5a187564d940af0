"""Verbatim pulls on the H100: scaled fp8 handles moved into scaled fp8 destinations of the same granularity by the
copy plan alone, bytes and scales compared as uint8 / uint32 with the group-by-group oracle over the layout table;
data a requantising pull would change (max |q| < 448, UE8M0, NaN / Inf groups, scales outside [2^-22, 2^119],
subnormal scales); source-side quantisation followed by a verbatim pull and refresh replays; dequantising from
the destination; one mixed pull; the errors; the state-dict API; peer mappings and the full-size Llama-3-8B
linear weights."""

import numpy as np
import pytest
import torch

import torchstore_b200 as ts
import workloads
from oracle.dequant_fp8_oracle import torch_dequantize
from oracle.verbatim_fp8_oracle import verbatim
from tests.helpers import (DEV, E4M3, cleanup, guards_intact, native_session, needs_two_gpus, pull_box, register_shards,
                           run)
from tests.test_verbatim_fp8_cpu import GRANULARITIES, KW, LAYOUTS, fp8_full, make_sources, rows
from torchstore_b200 import _native
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource, source_scale_shapes
from torchstore_b200.transport.types import TensorSlice

pytestmark = pytest.mark.gpu
_init = pytest.fixture(scope="module", autouse=True)(native_session)


def assert_oracle(g, sources, box, q, s):
    want_q, want_s, group = verbatim(g, [(sh.view(torch.uint8).numpy(), sc.numpy(), off) for sh, sc, off in sources], *box)
    assert group is None
    assert np.array_equal(q.view(torch.uint8).cpu().numpy(), want_q)
    assert np.array_equal(s.cpu().numpy().reshape(-1).view(np.uint32), want_s.reshape(-1).view(np.uint32))


@pytest.mark.parametrize("g", GRANULARITIES)
def test_layout_table_bit_exact(g):
    """Every layout of the table whose groups line up for `g`, through the copy plan alone."""
    ran = 0
    for name, gshape, boxes, box, lines_up in LAYOUTS:
        if g not in lines_up:
            continue
        sources = make_sources(g, fp8_full(gshape, len(name)), boxes, len(name) + 1)
        dev_sources, handles = register_shards(gshape, [(off, sh, sc) for sh, sc, off in sources], granularity=g)
        sync, q, s, bases = pull_box(handles, gshape, box, E4M3, granularity=g, verbatim=True)
        assert sync._native_plans and not any(sync._fp8_plans), name
        assert_oracle(g, sources, box, q, s)
        assert all(guards_intact(b) for b in bases), name
        sync.close()
        cleanup(dev_sources)
        ran += 1
    assert ran >= 7


# source scales a requantising pull would not keep: UE8M0 powers of two, outside [2^-22, 2^119], subnormal, Inf, NaN
SCALES = np.array([2.0 ** -7, 2.0 ** 3, 2.0 ** -30, 2.0 ** 125, 1e-40, 1.4e-45, np.inf, np.nan, -0.75, 0.0], np.float32)


def hard_sources(g):
    """A [2, 256, 512] stack in two row shards of 128 rows; every e4m3fn byte (NaN 0x7F / 0xFF included) in
    every row, rows whose max |q| is far below 448, and every shard's scales drawn from SCALES."""
    q = torch.arange(256, dtype=torch.uint8).repeat(2, 256, 2)
    q[:, ::3] &= 0x9F  # max |q| well under 448 on these rows
    q = q.view(E4M3)
    rng = np.random.default_rng(len(g))
    sources = []
    for off, loc in rows((2, 256, 512), 2, 0, 1):
        shard = q[:, off[1]: off[1] + loc[1]].contiguous()
        scale = rng.choice(SCALES, size=source_scale_shapes(g, loc, off[-2], off[-1])[0]).astype(np.float32)
        sources.append((shard, torch.from_numpy(scale), off))
    return sources


@pytest.mark.parametrize("g", GRANULARITIES)
def test_data_a_requantising_pull_would_change(g):
    sources = hard_sources(g)
    dev_sources, handles = register_shards((2, 256, 512), [(off, sh, sc) for sh, sc, off in sources], granularity=g)
    box = ((0, 128, 0), (2, 128, 512)) if g == "tensor" else ((0, 0, 256), (2, 256, 256))
    sync, q, s, bases = pull_box(handles, (2, 256, 512), box, E4M3, granularity=g, verbatim=True)
    assert_oracle(g, sources, box, q, s)
    # f32(q_dst) * s_dst is the source's, bit for bit: the dequantised values of both sides agree
    want = torch_dequantize(q, s, g, 0, 0, torch.float32)
    full_q = torch.cat([sh for sh, _, _ in sources], dim=1).to(DEV)
    region = full_q[tuple(slice(o, o + e) for o, e in zip(*box))]
    src_vals = torch.cat([torch_dequantize(sh.to(DEV), sc.to(DEV), g, off[-2], off[-1], torch.float32)
                          for sh, sc, off in sources], dim=1)[tuple(slice(o, o + e) for o, e in zip(*box))]
    assert torch.equal(q.view(torch.uint8), region.view(torch.uint8))
    assert torch.equal(want.view(torch.int32), src_vals.view(torch.int32))
    assert all(guards_intact(b) for b in bases)
    sync.close()
    cleanup(dev_sources)


@pytest.mark.parametrize("scale_fmt", [None, "ue8m0"])
@pytest.mark.parametrize("g", GRANULARITIES)
def test_source_quantised_chain_and_refresh(g, scale_fmt):
    """register(quantize=g) then a verbatim pull: the destination holds the source's staging bytes and scales;
    refresh() and a second pull replay the same plan and deliver the new bytes."""
    gshape = (512, 384)
    gen = torch.Generator(DEV).manual_seed(11)
    master = torch.randn(gshape, device=DEV, generator=gen).to(torch.bfloat16)
    srcs, handles = [], []
    for r, (off, loc) in enumerate(rows(gshape, 4)):
        src = DirectWeightSyncSource()
        w = master[off[0]: off[0] + loc[0]].clone()
        sl = TensorSlice(off, (r,), gshape, loc, (4,))
        handles.append(src.register({"w": w}, rank=r, tensor_slices={"w": sl}, quantize={"w": g}, scale_fmt=scale_fmt)["w"])
        srcs.append((src, w, off))
    box = rows(gshape, 4)[2] if g == "tensor" else ((0, 128), (512, 256))
    q = torch.zeros(box[1], dtype=E4M3, device=DEV)
    s = torch.zeros(source_scale_shapes(g, box[1], 0, 0)[0], device=DEV)
    sync = DirectWeightSyncDest()
    for step in range(2):
        run(sync.pull({"w": handles}, {"w": q}, {"w": TensorSlice(box[0], (0,), gshape, box[1], (1,))},
                      **{KW[g]: {"w": s}}, verbatim=True))
        if step == 0:
            ids = dict(sync._native_plans)
        else:
            assert dict(sync._native_plans) == ids  # replayed, not rebuilt
        staged = [(src._quantized["w"][0].cpu(), src._quantized["w"][1].cpu(), off) for src, _, off in srcs]
        assert_oracle(g, staged, box, q, s)
        for src, w, _ in srcs:
            w.mul_(-3)
            src.refresh()
    sync.close()
    for src, *_ in srcs:
        run(src.cleanup())


@pytest.mark.parametrize("g", GRANULARITIES)
def test_dequantising_from_the_destination_equals_the_source(g):
    gshape = (384, 512)
    sources = make_sources(g, fp8_full(gshape, 21), rows(gshape, 3), 22)
    dev_sources, handles = register_shards(gshape, [(off, sh, sc) for sh, sc, off in sources], granularity=g)
    box = ((128, 0), (128, 512)) if g == "tensor" else ((0, 256), (384, 256))
    sync, q, s, _ = pull_box(handles, gshape, box, E4M3, granularity=g, verbatim=True)
    from_dest = torch.zeros(box[1], device=DEV)
    back = DirectWeightSyncSource()
    h = back.register({"w": q}, rank=0, tensor_slices={"w": TensorSlice(box[0], (0,), gshape, box[1], (1,))},
                      **{KW[g]: {"w": s}})
    dsl = {"w": TensorSlice(box[0], (0,), gshape, box[1], (1,))}
    run(DirectWeightSyncDest().pull({"w": [h["w"]]}, {"w": from_dest}, dsl))
    from_src = torch.zeros(box[1], device=DEV)
    run(DirectWeightSyncDest().pull({"w": handles}, {"w": from_src}, dsl))
    assert torch.equal(from_dest.view(torch.int32), from_src.view(torch.int32))
    sync.close()
    run(back.cleanup())
    cleanup(dev_sources)


def test_mixed_pull_replay_and_rebuild():
    """Plain, cast, quantising, dequantising and verbatim names in one pull; replays, a flipped flag rebuilds, and
    a verbatim-only pull is one copy plan per device."""
    gshape = (256, 384)
    vb_sources = make_sources("block", fp8_full(gshape, 31), rows(gshape, 2), 32)
    dq_sources = make_sources("channel", fp8_full(gshape, 33), rows(gshape, 2), 34)
    vb_dev, vb_handles = register_shards(gshape, [(off, sh, sc) for sh, sc, off in vb_sources], granularity="block",
                                         name="vb")
    dq_dev, dq_handles = register_shards(gshape, [(off, sh, sc) for sh, sc, off in dq_sources], granularity="channel",
                                         name="dq")
    plain = (torch.randn(128, 64) * 0.1).to(torch.bfloat16)
    cast = torch.randn(128, 96) * 0.1
    master = (torch.randn(256, 256) * 0.1).to(torch.bfloat16)
    src = DirectWeightSyncSource()
    h = src.register({"plain": plain.to(DEV), "cast": cast.to(DEV), "quant": master.to(DEV)}, rank=0)
    dest = {"vb": torch.zeros(gshape, dtype=E4M3, device=DEV), "dq": torch.zeros(gshape, dtype=torch.bfloat16, device=DEV),
            "plain": torch.zeros(128, 64, dtype=torch.bfloat16, device=DEV),
            "cast": torch.zeros(128, 96, dtype=torch.bfloat16, device=DEV),
            "quant": torch.zeros(256, 256, dtype=E4M3, device=DEV)}
    vs, qs = torch.zeros(2, 3, device=DEV), torch.zeros(256, 1, device=DEV)
    handles = {"vb": vb_handles, "dq": dq_handles, "plain": [h["plain"]], "cast": [h["cast"]], "quant": [h["quant"]]}
    kw = dict(block_scales={"vb": vs}, channel_scales={"quant": qs})
    sync = DirectWeightSyncDest()
    launches = []
    for _ in range(3):
        before = _native.launch_count()
        run(sync.pull(handles, dest, **kw, verbatim=True))
        launches.append(_native.launch_count() - before)
        plans = [dict(p) for p in (sync._native_plans, sync._scaled_plans, sync._dequant_plans)]
        assert all(plans) and not sync._requant_plans and not sync._block_plans
        assert_oracle("block", vb_sources, ((0, 0), gshape), dest["vb"], vs)
        full_dq = torch.cat([sh for sh, _, _ in dq_sources]).to(DEV)
        full_ds = torch.cat([sc.reshape(-1, 1) for _, sc, _ in dq_sources]).to(DEV)
        torch.testing.assert_close(dest["dq"], torch_dequantize(full_dq, full_ds, "channel", 0, 0, torch.bfloat16),
                                   rtol=0, atol=0, equal_nan=True)  # random bytes hold NaNs
        assert torch.equal(dest["plain"].cpu(), plain) and torch.equal(dest["cast"], cast.to(DEV).to(torch.bfloat16))
    assert launches[1] == launches[2]
    first = plans
    run(sync.pull(handles, dest, **kw, verbatim=True))
    assert [dict(p) for p in (sync._native_plans, sync._scaled_plans, sync._dequant_plans)] == first
    # flipping the flag rebuilds, even where nothing is verbatim; without it the fp8 handles of 'vb' are refused
    sub = {k: dest[k] for k in ("plain", "quant")}
    run(sync.pull(handles, sub, channel_scales={"quant": qs}))
    ids = dict(sync._scaled_plans)
    run(sync.pull(handles, sub, channel_scales={"quant": qs}, verbatim=True))
    assert dict(sync._scaled_plans) != ids
    with pytest.raises(TypeError, match="requantised only with requantize=True"):
        run(sync.pull(handles, dest, **kw))
    # a verbatim-only pull: no fp8 plan, one kernel time per device
    only = DirectWeightSyncDest()
    vs.zero_()
    dest["vb"].zero_()
    run(only.pull({"vb": vb_handles}, {"vb": dest["vb"]}, block_scales={"vb": vs}, verbatim=True))
    assert not any(only._fp8_plans) and list(only.last_pull_ms) == [0]
    assert_oracle("block", vb_sources, ((0, 0), gshape), dest["vb"], vs)
    only.close()
    sync.close()
    cleanup(vb_dev)
    cleanup(dq_dev)
    run(src.cleanup())


def test_errors_raise_before_anything_is_compiled():
    gshape = (256, 768)
    q_full = fp8_full(gshape, 41)
    sources = make_sources("block", q_full, rows(gshape, 2) + [((64, 0), (128, 768))], 42)
    dev_sources, all_handles = register_shards(gshape, [(off, sh, sc) for sh, sc, off in sources], granularity="block")
    handles, overlapping = all_handles[:2], all_handles[2]
    bf16 = DirectWeightSyncSource()
    hb = bf16.register({"w": torch.zeros(256, 768, dtype=torch.bfloat16, device=DEV)}, rank=0)["w"]
    unscaled = DirectWeightSyncSource()
    hu = unscaled.register({"w": torch.zeros(256, 768, dtype=E4M3, device=DEV)}, rank=0)["w"]
    box = rows(gshape, 4, 1)[1]  # TP(4) columns 192..384: blocks straddle 256
    full = ((0, 0), gshape)

    def refuses(exc, match, hs, box, g="block", **kw):
        before = _native.launch_count()
        sync = DirectWeightSyncDest()
        with pytest.raises(exc, match=match):
            pull_box(hs, gshape, box, E4M3, granularity=g, sync=sync, verbatim=True, **kw)
        assert _native.launch_count() == before and sync._plan is None and not sync._native_plans

    refuses(ValueError, r"verbatim pull of 'w' \(block_scales\): destination block \(0, 0\).*requantize=True", handles, box)
    refuses(ValueError, "covered by no handle", handles[:1], full)
    refuses(ValueError, r"global element \(64, 0\) is covered by two handles", handles + [overlapping], full)
    refuses(ValueError, "channel destination|granularity only; use requantize=True", handles, full, "channel")
    refuses(ValueError, "exclusive", handles, full, requantize=True)
    refuses(ValueError, "scale_fmt does nothing here", handles, full, scale_fmt="ue8m0")
    refuses(TypeError, r"mix scaled fp8 and unscaled sources \(verbatim=True\)", handles + [hb], full)
    refuses(TypeError, "verbatim=True reads scaled fp8 handles", [hu], full)
    run(bf16.cleanup())
    run(unscaled.cleanup())
    cleanup(dev_sources)


def test_put_and_get_state_dict_verbatim():
    import torch.distributed as dist
    from torch.testing._internal.distributed.fake_pg import FakeStore

    from torchstore_b200 import state_dict_utils

    async def main():
        dist.init_process_group("fake", store=FakeStore(), rank=0, world_size=1)
        await ts.initialize()
        try:
            w = (torch.randn(256, 384, device=DEV) * 0.02).to(torch.bfloat16)
            await ts.put_state_dict({"w": w}, "policy_vb", direct_rdma=True, quantize={"w": "block"})
            src = state_dict_utils._get_rdma_cache(await ts.client()).sources["policy_vb"]
            dst = {"w": torch.zeros(256, 384, dtype=E4M3, device=DEV)}
            bs = torch.zeros(2, 3, device=DEV)
            for _ in range(2):
                out = await ts.get_state_dict("policy_vb", user_state_dict=dst, direct_rdma=True, block_scales={"w": bs},
                                              verbatim=True)
                assert out is dst
                q, s, _ = src._quantized["w"]
                assert torch.equal(dst["w"].view(torch.uint8), q.view(torch.uint8))
                assert torch.equal(bs.view(torch.int32), s.view(torch.int32))
                w.mul_(2)
                await ts.put_state_dict(None, "policy_vb", direct_rdma=True)
            with pytest.raises(NotImplementedError, match="verbatim"):
                await ts.get_state_dict("policy_vb", user_state_dict=dst, verbatim=True)
        finally:
            await ts.shutdown()
            dist.destroy_process_group()

    run(main())


@needs_two_gpus
@pytest.mark.parametrize("g", GRANULARITIES)
def test_weight_and_scale_read_over_peer_mappings(g):
    gshape = (512, 512)
    sources = make_sources(g, fp8_full(gshape, 51), rows(gshape, 4), 52)
    dev_sources, handles = [], []
    for r, sh in enumerate(sources):  # shards alternate between cuda:1 and cuda:0
        d, h = register_shards(gshape, [(off, sh, sc) for sh, sc, off in [sh]], granularity=g,
                               device=f"cuda:{1 - r % 2}")
        dev_sources += d
        handles += h
    box = rows(gshape, 4)[1] if g == "tensor" else ((0, 256), (512, 256))
    sync, q, s, bases = pull_box(handles, gshape, box, E4M3, granularity=g, verbatim=True)
    assert _native.plan_info(sync._native_plans[0]).remote_src_bytes > 0
    assert_oracle(g, sources, box, q, s)
    assert all(guards_intact(b) for b in bases)
    sync.close()
    cleanup(dev_sources)


def test_full_size_llama3_8b_linear_weights():
    """One layer's Llama-3-8B linear weights, block-quantised on the source in FSDP(8) row shards on one GPU and
    pulled verbatim into the TP(8) rank-3 shards (column- and row-parallel): bit-exact bytes and scales."""
    layout = {k.split(".")[-2]: v for k, v in workloads.llama_layout(n_layers=1, with_embeddings=False).items()
              if k.split(".")[-2] in ("wq", "wk", "wv", "wo", "w1", "w2", "w3")}
    gen = torch.Generator(DEV).manual_seed(7)
    srcs, handles, full_q, full_s = [], {}, {}, {}
    for name, (shape, _) in layout.items():
        master = (torch.randn(shape, device=DEV, generator=gen) * 0.02).to(torch.bfloat16)
        handles[name], qs, ss = [], [], []
        for r, (off, loc) in enumerate(rows(shape, 8)):
            src = DirectWeightSyncSource()
            w = master[off[0]: off[0] + loc[0]].clone()
            sl = TensorSlice(off, (r,), shape, loc, (8,))
            handles[name].append(src.register({name: w}, rank=r, tensor_slices={name: sl}, quantize={name: "block"})[name])
            qs.append(src._quantized[name][0])
            ss.append(src._quantized[name][1])
            srcs.append(src)
        full_q[name], full_s[name] = torch.cat(qs), torch.cat(ss)
        del master
    dest, scales, slices, boxes = {}, {}, {}, {}
    for name, (shape, (_, dim)) in layout.items():
        off, loc = rows(shape, 8, dim)[3]
        boxes[name] = (off, loc)
        dest[name] = torch.empty(loc, dtype=E4M3, device=DEV)
        scales[name] = torch.full(source_scale_shapes("block", loc, 0, 0)[0], -1.0, device=DEV)
        slices[name] = TensorSlice(off, (3,), shape, loc, (8,))
    sync = DirectWeightSyncDest()
    run(sync.pull(handles, dest, slices, block_scales=scales, verbatim=True))
    assert not any(sync._fp8_plans)
    for name, (off, loc) in boxes.items():
        want_q = full_q[name][off[0]: off[0] + loc[0], off[1]: off[1] + loc[1]]
        want_s = full_s[name][off[0] // 128: -(-(off[0] + loc[0]) // 128), off[1] // 128: -(-(off[1] + loc[1]) // 128)]
        assert torch.equal(dest[name].view(torch.uint8), want_q.view(torch.uint8)), name
        assert torch.equal(scales[name].view(torch.int32), want_s.view(torch.int32)), name
    sync.close()
    for src in srcs:
        run(src.cleanup())

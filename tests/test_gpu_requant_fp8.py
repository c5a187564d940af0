"""Requantising pulls on the H100: block-, channel- and tensor-scaled fp8 handles into block-, channel- and
tensor-scaled fp8 destinations, bit-exact against the numpy composition oracle and against the torch CUDA
composition (dequantise into f32, then quantise) with NaN bytes included, and byte for byte against the
two-step product route (a dequantising pull into an f32 temporary, then a quantising pull from it); guard
bytes, aligned identity, a mixed pull with replay and rebuild, the state-dict API, peer-mapped sources and a
full-size Llama-3-8B w1."""

from functools import partial

import numpy as np
import pytest
import torch

import torchstore_b200 as ts
from oracle.dequant_fp8_oracle import GRANULARITIES, SCALE_SET, scale_shape, torch_dequantize
from oracle.requant_fp8_oracle import PAIRS, quantize, torch_requantize
from tests.fp8_regimes import assert_requant_oracle, assert_requant_torch_cuda
from tests.helpers import (DEV, E4M3, KW, cleanup, dest_scale_shape, guards_intact, native_session, needs_two_gpus,
                           pull_box, register_boxes, run, shard_box)
from tests.test_dequant_fp8_cpu import local_scale as dq_local_scale
from tests.test_requant_fp8_cpu import fp8_full, global_scale
from torchstore_b200 import _native
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource
from torchstore_b200.transport.types import TensorSlice

pytestmark = pytest.mark.gpu
_init = pytest.fixture(scope="module", autouse=True)(native_session)


@pytest.mark.parametrize("sg,dg", PAIRS)
def test_reshard_matrix(sg, dg):
    """FSDP(6) row shards starting mid-block into row- and column-parallel TP destinations (350 rows / 260
    columns each: not 128-aligned)."""
    q = fp8_full((700, 520), 31)
    s = global_scale(sg, q.shape, 31)
    sources, handles = register_boxes(q, [shard_box(q.shape, 6, r, 0) for r in range(6)], granularity=sg,
                                      scale_of=partial(dq_local_scale, s, sg))
    for dst_dim in (0, 1):
        for d in range(2):
            box = shard_box(q.shape, 2, d, dst_dim)
            sync, y, ys, bases = pull_box(handles, q.shape, box, E4M3, granularity=dg, requantize=True)
            assert sync._requant_plans and not (sync._dequant_plans or sync._block_plans or sync._scaled_plans)
            assert_requant_oracle(y, ys, q, s, sg, box, dg)
            assert_requant_torch_cuda(y, ys, q, s, sg, box, dg)
            assert all(guards_intact(b) for b in bases)
            sync.close()
    cleanup(sources)


def scale_set_input(sg):
    """Every e4m3fn byte in every row, under a source scale set with 0, a negative scale, Inf and NaN."""
    scales = torch.from_numpy(SCALE_SET.copy())
    if sg == "block":
        q = torch.arange(256, dtype=torch.uint8).repeat(3 * 256, 1).view(3, 256, 256)
        return q.view(E4M3), scales.reshape(3, 2, 2)
    if sg == "channel":
        q = torch.arange(256, dtype=torch.uint8).repeat(len(SCALE_SET) * 16, 1)
        return q.view(E4M3), scales.repeat_interleave(16).reshape(-1, 1)
    q = torch.arange(256, dtype=torch.uint8).repeat(len(SCALE_SET) * 16, 1).view(len(SCALE_SET), 16, 256)
    return q.view(E4M3), scales


@pytest.mark.parametrize("sg,dg", PAIRS)
def test_differential_against_the_two_step_route(sg, dg):
    """The fused pull equals a dequantising pull into an f32 temporary followed by a quantising pull from it,
    fp8 bytes and scale_inv byte for byte, on fixture-like data and on the SCALE_SET inputs."""
    for q, s in (scale_set_input(sg), (fp8_full((3, 300, 260), 41), None)):
        s = s if s is not None else global_scale(sg, q.shape, 41)
        box = ((0,) * q.dim(), tuple(q.shape))
        sources, handles = register_boxes(q, [box], granularity=sg, scale_of=partial(dq_local_scale, s, sg))
        sync, y, ys, _ = pull_box(handles, q.shape, box, E4M3, granularity=dg, requantize=True)
        tmp = torch.zeros(q.shape, device=DEV)
        run(DirectWeightSyncDest().pull({"w": handles}, {"w": tmp}))  # dequantising pull into f32
        back = DirectWeightSyncSource()
        h = back.register({"w": tmp}, rank=0)
        y2 = torch.zeros(q.shape, dtype=E4M3, device=DEV)
        ys2 = torch.zeros(dest_scale_shape(dg, tuple(q.shape)), device=DEV)
        run(DirectWeightSyncDest().pull({"w": [h["w"]]}, {"w": y2}, **{KW[dg]: {"w": ys2}}))  # quantising pull
        assert torch.equal(y.view(torch.uint8), y2.view(torch.uint8))
        assert torch.equal(ys.view(torch.int32), ys2.view(torch.int32))
        assert_requant_torch_cuda(y, ys, q, s, sg, box, dg)
        sync.close()
        run(back.cleanup())
        cleanup(sources)


@pytest.mark.parametrize("g", GRANULARITIES)
def test_aligned_identity(g):
    """Formula-quantised finite data, same granularity and aligned groups: the fp8 bytes come back unchanged."""
    x = torch.randn(2, 512, 768, generator=torch.Generator().manual_seed(4)) * 3
    q_np, s_np = quantize(x.numpy(), g)
    q = torch.from_numpy(q_np).view(E4M3)
    s = torch.from_numpy(np.asarray(s_np, np.float32).copy()).reshape(scale_shape(g, q.shape))
    sources, handles = register_boxes(q, [shard_box(q.shape, 4, r, 1) for r in range(4)], granularity=g,
                                      scale_of=partial(dq_local_scale, s, g))
    sync, y, ys, _ = pull_box(handles, q.shape, ((0, 0, 0), tuple(q.shape)), E4M3, granularity=g, requantize=True)
    assert torch.equal(y.view(torch.uint8).cpu(), q.view(torch.uint8))
    sync.close()
    cleanup(sources)


def test_mixed_pull_replay_and_rebuild():
    """One pull holds plain, cast, quantising, dequantising and requantising names; a second pull replays with
    no rebuild; a new scale dict or a flipped requantize rebuilds."""
    q = fp8_full((300, 260), 51)
    s = global_scale("block", q.shape, 51)
    dq_sources, dq_handles = register_boxes(q, [shard_box(q.shape, 3, r, 0) for r in range(3)], granularity="block",
                                            scale_of=partial(dq_local_scale, s, "block"), name="dq")
    rq_sources, rq_handles = register_boxes(q, [shard_box(q.shape, 3, r, 0) for r in range(3)], granularity="block",
                                            scale_of=partial(dq_local_scale, s, "block"), name="rq")
    plain = (torch.randn(128, 64) * 0.1).to(torch.bfloat16)
    cast = (torch.randn(128, 96) * 0.1)
    master = (torch.randn(256, 256) * 0.1).to(torch.bfloat16)
    src = DirectWeightSyncSource()
    h = src.register({"plain": plain.to(DEV), "cast": cast.to(DEV), "quant": master.to(DEV)}, rank=0)
    dest = {"dq": torch.zeros(300, 260, dtype=torch.bfloat16, device=DEV),
            "rq": torch.zeros(300, 260, dtype=E4M3, device=DEV),
            "plain": torch.zeros(128, 64, dtype=torch.bfloat16, device=DEV),
            "cast": torch.zeros(128, 96, dtype=torch.bfloat16, device=DEV),
            "quant": torch.zeros(256, 256, dtype=E4M3, device=DEV)}
    bs, cs = torch.zeros(2, 2, device=DEV), torch.zeros(300, 1, device=DEV)
    handles = {"dq": dq_handles, "rq": rq_handles, "plain": [h["plain"]], "cast": [h["cast"]], "quant": [h["quant"]]}
    sync = DirectWeightSyncDest()
    kw = dict(block_scales={"quant": bs}, channel_scales={"rq": cs})
    launches = []
    for _ in range(3):
        before = _native.launch_count()
        run(sync.pull(handles, dest, **kw, requantize=True))
        launches.append(_native.launch_count() - before)
        plans = [dict(p) for p in (sync._native_plans, sync._block_plans, sync._dequant_plans, sync._requant_plans)]
        assert all(plans)
        assert torch.equal(dest["dq"], torch_dequantize(q.to(DEV), s.to(DEV), "block"))
        want_q, want_s = torch_requantize(q.to(DEV), s.to(DEV), "block", 0, 0, "channel")
        assert torch.equal(dest["rq"].view(torch.uint8), want_q.view(torch.uint8)) and torch.equal(cs, want_s)
        assert torch.equal(dest["plain"].cpu(), plain) and torch.equal(dest["cast"], cast.to(DEV).to(torch.bfloat16))
    assert launches[1] == launches[2]  # replays launch the same kernels
    first = plans
    run(sync.pull(handles, dest, **kw, requantize=True))
    assert [dict(p) for p in (sync._native_plans, sync._block_plans, sync._dequant_plans, sync._requant_plans)] == first
    cs2 = torch.zeros(300, 1, device=DEV)  # a new scale dict: rebuilt
    run(sync.pull(handles, dest, block_scales={"quant": bs}, channel_scales={"rq": cs2}, requantize=True))
    assert dict(sync._requant_plans) != first[3] and torch.equal(cs2, cs)
    # flipping the flag rebuilds even where nothing is requantised
    sub = {k: dest[k] for k in ("plain", "quant")}
    run(sync.pull(handles, sub, block_scales={"quant": bs}))
    ids = dict(sync._block_plans)
    run(sync.pull(handles, sub, block_scales={"quant": bs}, requantize=True))
    assert dict(sync._block_plans) != ids and not sync._requant_plans
    # a destination group the handles do not cover: ValueError naming it, before any launch
    before = _native.launch_count()
    part = {"rq": torch.zeros(400, 260, dtype=E4M3, device=DEV)}
    with pytest.raises(ValueError, match="requantising pull of 'rq'.*group"):
        run(DirectWeightSyncDest().pull({"rq": rq_handles}, part, {"rq": TensorSlice((0, 0), (0,), (400, 260), (400, 260), (1,))},
                                        channel_scales={"rq": torch.zeros(400, 1, device=DEV)}, requantize=True))
    assert _native.launch_count() == before
    sync.close()
    cleanup(dq_sources)
    cleanup(rq_sources)
    run(src.cleanup())


def test_put_and_get_state_dict_requantise():
    import torch.distributed as dist
    from torch.testing._internal.distributed.fake_pg import FakeStore

    async def main():
        dist.init_process_group("fake", store=FakeStore(), rank=0, world_size=1)
        await ts.initialize()
        try:
            q = fp8_full((256, 384), 61).to(DEV)
            sb = global_scale("block", q.shape, 61).to(DEV)
            await ts.put_state_dict({"w": q}, "policy_rq", direct_rdma=True, block_scales={"w": sb})
            dst = {"w": torch.zeros(256, 384, dtype=E4M3, device=DEV)}
            cs = torch.zeros(256, 1, device=DEV)
            for _ in range(2):
                out = await ts.get_state_dict("policy_rq", user_state_dict=dst, direct_rdma=True, channel_scales={"w": cs},
                                              requantize=True)
                assert out is dst
                want_q, want_s = torch_requantize(q, sb, "block", 0, 0, "channel")
                assert torch.equal(dst["w"].view(torch.uint8), want_q.view(torch.uint8)) and torch.equal(cs, want_s)
                sb.mul_(0.5)
                await ts.put_state_dict(None, "policy_rq", direct_rdma=True)
            with pytest.raises(NotImplementedError):
                await ts.get_state_dict("policy_rq", user_state_dict=dst, requantize=True)
        finally:
            await ts.shutdown()
            dist.destroy_process_group()

    run(main())


@needs_two_gpus
@pytest.mark.parametrize("sg,dg", [("block", "channel"), ("channel", "block"), ("tensor", "tensor")])
def test_weight_and_scale_read_over_peer_mappings(sg, dg):
    q = fp8_full((300, 520), 71)
    s = global_scale(sg, q.shape, 71)
    sources, handles = [], []
    for r, b in enumerate([shard_box(q.shape, 4, r, 0) for r in range(4)]):  # shards alternate between cuda:1 and cuda:0
        s_, h_ = register_boxes(q, [b], granularity=sg, scale_of=partial(dq_local_scale, s, sg),
                                device=f"cuda:{1 - r % 2}")
        sources += s_
        handles += h_
    for d in range(2):
        box = shard_box(q.shape, 2, d, 1)
        sync, y, ys, bases = pull_box(handles, q.shape, box, E4M3, granularity=dg, requantize=True)
        assert _native.plan_info(sync._requant_plans[0]).remote_src_bytes > 0
        assert_requant_torch_cuda(y, ys, q, s, sg, box, dg)
        assert all(guards_intact(b) for b in bases)
        sync.close()
    cleanup(sources)


def test_full_size_llama3_8b_w1():
    """Llama-3-8B w1 [14336, 4096] from 6 block-scaled FSDP row shards (boundaries mid-block) into a per-channel
    destination, against the torch CUDA composition."""
    rows, cols = 14336, 4096
    x = torch.randn(rows, cols, device=DEV, generator=torch.Generator(DEV).manual_seed(5)) * 0.02
    from oracle.block_fp8_oracle import torch_quantize

    q, s = torch_quantize(x)
    del x
    boxes = [shard_box((rows, cols), 6, r, 0) for r in range(6)]
    sources, handles = register_boxes(q, boxes, granularity="block", scale_of=partial(dq_local_scale, s, "block"))
    sync, y, ys, bases = pull_box(handles, (rows, cols), ((0, 0), (rows, cols)), E4M3, granularity="channel",
                                  requantize=True)
    want_q, want_s = torch_requantize(q, s, "block", 0, 0, "channel")
    assert torch.equal(y.view(torch.uint8), want_q.view(torch.uint8)) and torch.equal(ys, want_s)
    assert all(guards_intact(b) for b in bases)
    sync.close()
    cleanup(sources)

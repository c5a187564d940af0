"""Dequantising pulls on the H100: block-, channel- and tensor-scaled fp8 handles into bf16 / f16 / f32
destinations, bit-exact against the numpy oracle on every non-NaN output and against the torch CUDA
rendering (q.float() * s).to(dst) with NaN bytes included; guard bytes, mixed pulls, plan replay and
rebuild, the state-dict API, the quantise -> dequantise round trip and peer-mapped sources."""

from functools import partial

import numpy as np
import pytest
import torch

import torchstore_b200 as ts
from oracle.block_fp8_oracle import quantize as block_quantize
from oracle.dequant_fp8_oracle import GRANULARITIES, SCALE_SET, scale_shape, torch_dequantize
from tests.fp8_regimes import assert_dequant_oracle, assert_dequant_torch_cuda, want_bits
from tests.helpers import (DEV, E4M3, KW, cleanup, guards_intact, native_session, needs_two_gpus, pull_box, region,
                           register_boxes, run, shard_box)
from tests.test_dequant_fp8_cpu import fp8_full, global_scale, local_scale
from torchstore_b200 import _native
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource, ScaledNvlinkBuffer
from torchstore_b200.transport.types import TensorSlice

pytestmark = pytest.mark.gpu
DTYPES = [torch.bfloat16, torch.float16, torch.float32]
_init = pytest.fixture(scope="module", autouse=True)(native_session)


@pytest.mark.parametrize("g", GRANULARITIES)
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("n,dst_dim", [(6, 0), (3, 1)])
def test_fsdp_to_tp_reshard(g, dtype, n, dst_dim):
    """FSDP(n) shards starting mid-block into column- and row-parallel TP destinations."""
    q = fp8_full((700, 520), 10 * n + dst_dim)
    s = global_scale(g, q.shape, n)
    sources, handles = register_boxes(q, [shard_box(q.shape, n, r, 0) for r in range(n)], granularity=g,
                                      scale_of=partial(local_scale, s, g))
    for d in range(2):
        box = shard_box(q.shape, 2, d, dst_dim)
        sync, y, _, (base,) = pull_box(handles, q.shape, box, dtype)
        assert sync._dequant_plans and not sync._block_plans and not sync._scaled_plans
        assert_dequant_oracle(y, want_bits(q, s, g, box, dtype))
        assert_dequant_torch_cuda(y, q, s, g, box)
        assert guards_intact(base)
        sync.close()
    cleanup(sources)


@pytest.mark.parametrize("dtype", DTYPES)
def test_every_byte_against_the_scale_set(dtype):
    """All 256 e4m3fn bytes times 1, powers of two, amax/448, f32-subnormal products, f16 / bf16 overflow,
    0, a negative scale, Inf and NaN: torch CUDA bit for bit, NaN bytes included."""
    q = torch.arange(256, dtype=torch.uint8).repeat(len(SCALE_SET), 1).view(E4M3)
    s = torch.from_numpy(SCALE_SET.copy()).reshape(-1, 1)
    sources, handles = register_boxes(q, [((0, 0), tuple(q.shape))], granularity="channel",
                                      scale_of=partial(local_scale, s, "channel"))
    sync, y, _, (base,) = pull_box(handles, q.shape, ((0, 0), tuple(q.shape)), dtype)
    assert_dequant_torch_cuda(y, q, s, "channel", ((0, 0), tuple(q.shape)))
    assert_dequant_oracle(y, want_bits(q, s, "channel", ((0, 0), tuple(q.shape)), dtype))
    assert guards_intact(base)
    sync.close()
    cleanup(sources)


@pytest.mark.parametrize("g", GRANULARITIES)
def test_ep_moe_stack_and_replicas(g):
    q = fp8_full((4, 130, 260), 5)
    s = global_scale(g, q.shape, 5)
    boxes = [shard_box(q.shape, 2, r % 2, 0) for r in range(4)]  # EP(2) x replicated(2)
    sources, handles = register_boxes(q, boxes, granularity=g, scale_of=partial(local_scale, s, g))
    box = ((0, 0, 0), (4, 130, 260))
    sync, y, _, (base,) = pull_box(handles, q.shape, box, torch.bfloat16)
    assert_dequant_torch_cuda(y, q, s, g, box)
    sync.close()
    cleanup(sources)


def test_strided_windows_leave_the_rest_alone():
    """A destination window the handles cover only partly: uncovered elements keep their bytes."""
    q = fp8_full((256, 512), 7)
    s = global_scale("block", q.shape, 7)
    box = ((0, 0), (256, 384))
    sources, handles = register_boxes(q, [box], granularity="block",
                                      scale_of=partial(local_scale, s, "block"))  # columns 384.. are published by no handle
    dest = torch.full((256, 512), 3.0, dtype=torch.bfloat16, device=DEV)
    dsl = TensorSlice((0, 0), (0,), (256, 512), (256, 512), (1,))
    sync = DirectWeightSyncDest()
    run(sync.pull({"w": handles}, {"w": dest}, {"w": dsl}))
    assert torch.equal(dest[:, :384], torch_dequantize(region(q, *box).to(DEV), local_scale(s, "block", *box).to(DEV), "block"))
    assert bool((dest[:, 384:] == 3.0).all())
    sync.close()
    cleanup(sources)


def test_mixed_pull_dequant_plain_cast_and_quantise():
    """One pull: a block-dequantised name, a plain bf16 name, an unscaled fp8 -> bf16 cast and a block-quantising name."""
    q = fp8_full((300, 260), 9)
    s = global_scale("block", q.shape, 9)
    dq_sources, dq_handles = register_boxes(q, [shard_box(q.shape, 3, r, 0) for r in range(3)], granularity="block",
                                            scale_of=partial(local_scale, s, "block"), name="dq")
    plain = (torch.randn(128, 64) * 0.1).to(torch.bfloat16)
    raw = fp8_full((128, 96), 10)
    master = (torch.randn(256, 256) * 0.1).to(torch.bfloat16)
    src = DirectWeightSyncSource()
    h = src.register({"plain": plain.to(DEV), "raw": raw.to(DEV), "quant": master.to(DEV)}, rank=0)
    dest = {"dq": torch.zeros(300, 260, dtype=torch.bfloat16, device=DEV), "plain": torch.zeros(128, 64, dtype=torch.bfloat16, device=DEV),
            "raw": torch.zeros(128, 96, dtype=torch.bfloat16, device=DEV), "quant": torch.zeros(256, 256, dtype=E4M3, device=DEV)}
    bs = torch.zeros(2, 2, device=DEV)
    sync = DirectWeightSyncDest()
    handles = {"dq": dq_handles, "plain": [h["plain"]], "raw": [h["raw"]], "quant": [h["quant"]]}
    for _ in range(2):
        run(sync.pull(handles, dest, block_scales={"quant": bs}))
        assert torch.equal(dest["dq"], torch_dequantize(q.to(DEV), s.to(DEV), "block"))
        assert torch.equal(dest["plain"].cpu(), plain)
        assert torch.equal(dest["raw"], raw.to(DEV).to(torch.bfloat16))
        want_q, want_s = block_quantize(master.float().numpy())
        assert np.array_equal(dest["quant"].view(torch.uint8).cpu().numpy(), want_q)
        assert np.array_equal(bs.cpu().numpy().view(np.uint32), want_s.view(np.uint32))
    assert set(sync.last_pull_ms) == {0}
    sync.close()
    cleanup(dq_sources)
    run(src.cleanup())


def test_scaled_handles_never_take_the_unscaled_cast():
    """Regression: a scaled handle pulled into bf16 is dequantised, never cast as raw e4m3fn bytes."""
    q = fp8_full((128, 128), 11)
    s = torch.full((1, 1), 0.25)
    sources, handles = register_boxes(q, [((0, 0), (128, 128))], granularity="block",
                                      scale_of=partial(local_scale, s, "block"))
    sync, y, _, _ = pull_box(handles, q.shape, ((0, 0), (128, 128)), torch.bfloat16)
    assert not sync._native_plans and len(sync._dequant_plans) == 1
    assert torch.equal(y, (q.to(DEV).float() * 0.25).to(torch.bfloat16))
    assert not torch.equal(y, q.to(DEV).to(torch.bfloat16))
    # an fp8 destination gets the raw bytes
    q8 = torch.zeros(128, 128, dtype=E4M3, device=DEV)
    run(DirectWeightSyncDest().pull({"w": handles}, {"w": q8}))
    assert torch.equal(q8.view(torch.uint8).cpu(), q.view(torch.uint8))
    sync.close()
    cleanup(sources)


def test_replay_after_source_change_and_rebuild_after_destination_change():
    q = fp8_full((256, 256), 12)
    s = global_scale("channel", q.shape, 12)
    sources, handles = register_boxes(q, [shard_box(q.shape, 2, r, 0) for r in range(2)], granularity="channel",
                                      scale_of=partial(local_scale, s, "channel"))
    dest = {"w": torch.zeros(256, 256, dtype=torch.float16, device=DEV)}
    sync = DirectWeightSyncDest()
    run(sync.pull({"w": handles}, dest))
    plans = dict(sync._dequant_plans)
    for _, shard, scale in sources:  # new weights and scales in place: the cached plan reads them
        shard.copy_(fp8_full(tuple(shard.shape), 13).to(DEV))
        scale.mul_(2.0)
    run(sync.pull({"w": handles}, dest))
    assert dict(sync._dequant_plans) == plans
    q2 = torch.cat([shard.cpu() for _, shard, _ in sources])
    s2 = torch.cat([scale.cpu() for _, _, scale in sources])
    assert torch.equal(dest["w"], torch_dequantize(q2.to(DEV), s2.to(DEV), "channel", dst=torch.float16))
    dest["w"] = torch.zeros(256, 256, dtype=torch.float16, device=DEV)  # new destination memory: rebuilt
    run(sync.pull({"w": handles}, dest))
    assert dict(sync._dequant_plans) != plans
    assert torch.equal(dest["w"], torch_dequantize(q2.to(DEV), s2.to(DEV), "channel", dst=torch.float16))
    sync.close()
    cleanup(sources)


@pytest.mark.parametrize("g", GRANULARITIES)
def test_round_trip_through_the_quantising_pull(g):
    """bf16 -> (quantising pull) -> fp8 + scales -> registered as scaled handles -> (dequantising pull) -> bf16
    equals torch's dequant(quant(x))."""
    from oracle.scaled_fp8_oracle import torch_quantize

    x = (torch.randn(300, 260) * 0.05).to(torch.bfloat16)
    src = DirectWeightSyncSource()
    h = src.register({"w": x.to(DEV)}, rank=0)
    q = torch.zeros(300, 260, dtype=E4M3, device=DEV)
    sq = torch.zeros(scale_shape(g, (300, 260)), device=DEV)
    run(DirectWeightSyncDest().pull({"w": [h["w"]]}, {"w": q}, **{KW[g]: {"w": sq}}))
    back = DirectWeightSyncSource()
    hb = back.register({"w": q}, rank=0, **{KW[g]: {"w": sq}})
    y = torch.zeros(300, 260, dtype=torch.bfloat16, device=DEV)
    run(DirectWeightSyncDest().pull({"w": [hb["w"]]}, {"w": y}))
    if g == "block":
        from oracle.block_fp8_oracle import torch_quantize as block_torch_quantize

        tq, ts_ = block_torch_quantize(x.to(DEV))
    else:
        tq, ts_ = torch_quantize(x.to(DEV), g)
    assert torch.equal(y, torch_dequantize(tq, ts_, g))
    run(src.cleanup())
    run(back.cleanup())


def test_scaled_buffer_pickles_and_moves_raw_bytes():
    import pickle

    q = fp8_full((128, 256), 14).to(DEV)
    s = torch.ones(1, 2, device=DEV)
    src = DirectWeightSyncSource()
    h = src.register({"w": q}, rank=0, block_scales={"w": s})["w"]
    buf = pickle.loads(pickle.dumps(h.rdma_buffer))
    assert isinstance(buf, ScaledNvlinkBuffer) and buf.granularity == "block" and (buf.row0, buf.col0) == (0, 0)
    out = torch.zeros(q.numel(), dtype=torch.uint8, device=DEV)
    run(buf.read_into(out))
    assert torch.equal(out, q.view(torch.uint8).reshape(-1))
    run(src.cleanup())


def test_put_and_get_state_dict_with_scaled_sources():
    import torch.distributed as dist
    from torch.testing._internal.distributed.fake_pg import FakeStore

    async def main():
        dist.init_process_group("fake", store=FakeStore(), rank=0, world_size=1)
        await ts.initialize()
        try:
            q = fp8_full((256, 384), 15).to(DEV)
            sb = global_scale("block", q.shape, 15).to(DEV)
            sc = global_scale("channel", q.shape, 16).to(DEV)
            src = {"a": q, "b": q.clone(), "norm": torch.randn(384, device=DEV).to(torch.bfloat16)}
            await ts.put_state_dict(src, "policy_dq", direct_rdma=True, block_scales={"a": sb}, channel_scales={"b": sc})
            dst = {"a": torch.zeros(256, 384, dtype=torch.bfloat16, device=DEV), "b": torch.zeros(256, 384, device=DEV),
                   "norm": torch.zeros(384, dtype=torch.bfloat16, device=DEV)}
            for _ in range(2):
                out = await ts.get_state_dict("policy_dq", user_state_dict=dst, direct_rdma=True)
                assert out is dst
                assert torch.equal(dst["a"], torch_dequantize(src["a"], sb, "block"))
                assert torch.equal(dst["b"], torch_dequantize(src["b"], sc, "channel", dst=torch.float32))
                assert torch.equal(dst["norm"], src["norm"])
                sb.mul_(0.5)
                await ts.put_state_dict(None, "policy_dq", direct_rdma=True)
            with pytest.raises(NotImplementedError):
                await ts.put_state_dict(src, "policy_dq2", block_scales={"a": sb})
        finally:
            await ts.shutdown()
            dist.destroy_process_group()

    run(main())


def test_validation_raises_before_any_launch():
    q = fp8_full((256, 256), 17)
    s = global_scale("block", q.shape, 17)
    sources, handles = register_boxes(q, [((0, 0), (256, 256))], granularity="block",
                                      scale_of=partial(local_scale, s, "block"))
    psrc = DirectWeightSyncSource()
    plain = psrc.register({"w": q.to(DEV)}, rank=1)["w"]
    csources, chandles = register_boxes(q, [((0, 0), (256, 256))], granularity="channel",
                                        scale_of=partial(local_scale, global_scale("channel", q.shape, 1), "channel"))
    before = _native.launch_count()
    cases = [
        (ValueError, handles + [plain], torch.zeros(256, 256, dtype=torch.bfloat16, device=DEV)),
        (ValueError, handles + chandles, torch.zeros(256, 256, dtype=torch.bfloat16, device=DEV)),
        (TypeError, handles, torch.zeros(256, 256, dtype=torch.float64, device=DEV)),
        (TypeError, handles, torch.zeros(256, 256, dtype=torch.float8_e5m2, device=DEV)),
        (ValueError, handles, torch.zeros(256, 256, dtype=torch.bfloat16, device=DEV).t()),
    ]
    for exc, h, dest in cases:
        sync = DirectWeightSyncDest()
        with pytest.raises(exc, match="'w'"):
            run(sync.pull({"w": h}, {"w": dest}))
        assert not sync._dequant_plans and not sync._native_plans
    # a scaled destination fed by scaled handles: requantising is not offered
    with pytest.raises(TypeError):
        run(DirectWeightSyncDest().pull({"w": handles}, {"w": torch.zeros(256, 256, dtype=E4M3, device=DEV)},
                                        block_scales={"w": torch.zeros(2, 2, device=DEV)}))
    assert _native.launch_count() == before
    # register(): wrong scale shape / device / dtype and a DTensor-like refusal, nothing exported
    w = q.to(DEV)
    for exc, scale in ((ValueError, torch.zeros(3, 2, device=DEV)), (ValueError, torch.zeros(2, 2)),
                       (TypeError, torch.zeros(2, 2, device=DEV, dtype=torch.float64)), (TypeError, [1.0])):
        with pytest.raises(exc, match="'w'"):
            DirectWeightSyncSource().register({"w": w}, 0, block_scales={"w": scale})
    cleanup(sources)
    cleanup(csources)
    run(psrc.cleanup())


@needs_two_gpus
@pytest.mark.parametrize("g", GRANULARITIES)
def test_weight_and_scale_read_over_peer_mappings(g):
    q = fp8_full((300, 520), 18)
    s = global_scale(g, q.shape, 18)
    sources, handles = [], []
    for r, b in enumerate([shard_box(q.shape, 4, r, 0) for r in range(4)]):  # shards alternate between cuda:1 and cuda:0
        s_, h_ = register_boxes(q, [b], granularity=g, scale_of=partial(local_scale, s, g), device=f"cuda:{1 - r % 2}")
        sources += s_
        handles += h_
    for d in range(2):
        box = shard_box(q.shape, 2, d, 1)
        sync, y, _, (base,) = pull_box(handles, q.shape, box, torch.bfloat16)
        assert _native.plan_info(sync._dequant_plans[0]).remote_src_bytes > 0
        assert_dequant_torch_cuda(y, q, s, g, box)
        assert guards_intact(base)
        sync.close()
    cleanup(sources)

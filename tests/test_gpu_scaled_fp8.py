"""Per-channel and per-tensor scaled FP8 pulls on the H100: bf16/f16/f32 handles quantised into
float8_e4m3fn destinations with one float32 scale_inv per row or per matrix, during the gather.  Checked
bit for bit against the numpy oracle (finite data) and against a torch-CUDA tensor/tensor rendering of
the formula (special values, NaN bytes included); both kernel paths, reshards, mixed dicts, plan replay
and invalidation, the public state-dict API, validation before any launch, and peer-mapped sources on a
second GPU."""

import numpy as np
import pytest
import torch

import torchstore_b200 as ts
from oracle.block_fp8_oracle import quantize as block_quantize
from oracle.scaled_fp8_oracle import GRANULARITIES, quantize
from tests.helpers import (DEV, E4M3, cleanup, guards_intact, native_session, needs_two_gpus, pull_box, rand_full, region,
                           register_boxes, run, shard_box)
from tests.quant_pull_regimes import assert_scaled_torch_cuda
from tests.test_scaled_fp8_cpu import fixture_cases
from torchstore_b200 import _native
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource
from torchstore_b200.transport.types import TensorSlice

pytestmark = pytest.mark.gpu
_init = pytest.fixture(scope="module", autouse=True)(native_session)


def assert_oracle(q, s, x_f32, g):
    want_q, want_s = quantize(x_f32, g)
    assert np.array_equal(q.view(torch.uint8).cpu().numpy(), want_q)
    assert np.array_equal(s.cpu().numpy().view(np.uint32), want_s.view(np.uint32))


FINITE = [c for c in fixture_cases() if "nonfinite" not in c[0]]


@pytest.mark.parametrize("case", FINITE, ids=lambda c: c[0])
def test_exact_match_pull_of_the_fixture_shapes(case):
    _, g, dtype, x, _, _ = case
    full = torch.from_numpy(x).to(getattr(torch, dtype))
    shape = tuple(full.shape)
    sources, handles = register_boxes(full, [(tuple(0 for _ in shape), shape)])
    sync, q, s, (qb, sb) = pull_box(handles, shape, (tuple(0 for _ in shape), shape), E4M3, granularity=g)
    assert_oracle(q, s, x, g)
    assert guards_intact(qb) and guards_intact(sb)
    sync.close()
    cleanup(sources)


@pytest.mark.parametrize("case", [c for c in fixture_cases() if "nonfinite" in c[0] or "huge" in c[0] or "zero" in c[0]],
                         ids=lambda c: c[0])
def test_special_value_groups_match_torch_cuda_bit_for_bit(case):
    _, g, dtype, x, _, _ = case
    full = torch.from_numpy(x).to(getattr(torch, dtype))
    shape = tuple(full.shape)
    sources, handles = register_boxes(full, [((0, 0), shape)])
    sync, q, s, _ = pull_box(handles, shape, ((0, 0), shape), E4M3, granularity=g)
    assert_scaled_torch_cuda(q, s, full, g)
    sync.close()
    cleanup(sources)


@pytest.mark.parametrize("dtype,cols", [(torch.bfloat16, 4096), (torch.bfloat16, 14336), (torch.bfloat16, 16400),
                                        (torch.float32, 8192), (torch.float32, 8200), (torch.float16, 16401)])
def test_rows_inside_and_beyond_the_stage_bound(dtype, cols):
    """Rows of at most 32 KiB take the row-staged kernel, longer ones the two-pass one; 16401 is ragged."""
    full = rand_full((12, cols), dtype, cols)
    boxes = [shard_box(full.shape, 3, r, 1) for r in range(3)]  # unaligned column shards
    sources, handles = register_boxes(full, boxes)
    sync, q, s, (qb, sb) = pull_box(handles, full.shape, ((0, 0), tuple(full.shape)), E4M3, granularity="channel")
    info = _native.plan_info(sync._scaled_plans[0])
    staged = cols * full.element_size() <= 32768
    assert (info.num_tiles <= 12) == staged  # at most one band per row vs a tile per row and shard
    assert_oracle(q, s, full.float().numpy(), "channel")
    assert guards_intact(qb) and guards_intact(sb)
    sync.close()
    cleanup(sources)


@pytest.mark.parametrize("g", GRANULARITIES)
@pytest.mark.parametrize("n,dst_dim", [(4, 0), (4, 1), (3, 1)])
def test_fsdp_to_tp_reshard(g, n, dst_dim):
    full = rand_full((1000, 520), torch.bfloat16, 10 * n + dst_dim)  # per tensor: several tiles per shard
    sources, handles = register_boxes(full, [shard_box(full.shape, n, r, 0) for r in range(n)])
    for d in range(n):
        dst = shard_box(full.shape, n, d, dst_dim)
        sync, q, s, (qb, sb) = pull_box(handles, full.shape, dst, E4M3, granularity=g)
        assert_oracle(q, s, region(full, *dst).float().numpy(), g)
        assert guards_intact(qb) and guards_intact(sb)
        sync.close()
    cleanup(sources)


@pytest.mark.parametrize("g", GRANULARITIES)
def test_moe_stack(g):
    full = rand_full((3, 130, 260), torch.float32, 5)
    sources, handles = register_boxes(full, [shard_box(full.shape, 3, r, 1) for r in range(3)])
    for d in range(2):
        dst = shard_box(full.shape, 2, d, 2)
        sync, q, s, _ = pull_box(handles, full.shape, dst, E4M3, granularity=g)
        assert_oracle(q, s, region(full, *dst).float().numpy(), g)
        sync.close()
    cleanup(sources)


def test_per_tensor_scale_shapes_with_a_trailing_one():
    full = rand_full((2, 300, 200), torch.bfloat16, 9)
    sources, handles = register_boxes(full, [((0, 0, 0), (2, 300, 200))])
    q = torch.zeros(2, 300, 200, dtype=E4M3, device=DEV)
    s = torch.zeros(2, 1, device=DEV)  # compressed-tensors keeps [E, 1]; vLLM [E]
    sync = DirectWeightSyncDest()
    run(sync.pull({"w": handles}, {"w": q}, tensor_scales={"w": s}))
    assert_oracle(q, s.view(2), full.float().numpy(), "tensor")
    sync.close()
    cleanup(sources)


def test_mixed_dict_of_plain_block_channel_and_tensor_names():
    gen = torch.Generator().manual_seed(3)
    sd = {n: (torch.randn(256, 384, generator=gen) * 0.1).to(torch.bfloat16) for n in ("plain", "blk", "ch", "tn")}
    sd["byte"] = torch.randint(0, 255, (1000,), dtype=torch.uint8, generator=gen)
    src = DirectWeightSyncSource()
    handles = src.register({k: v.to(DEV) for k, v in sd.items()}, rank=0)
    dest = {"plain": torch.zeros(256, 384, dtype=torch.bfloat16, device=DEV), "byte": torch.zeros(1000, dtype=torch.uint8, device=DEV)}
    for n in ("blk", "ch", "tn"):
        dest[n] = torch.zeros(256, 384, dtype=E4M3, device=DEV)
    bs, cs, tsc = torch.zeros(2, 3, device=DEV), torch.zeros(256, 1, device=DEV), torch.zeros((), device=DEV)
    sync = DirectWeightSyncDest()
    run(sync.pull({k: [h] for k, h in handles.items()}, dest, block_scales={"blk": bs}, channel_scales={"ch": cs},
                  tensor_scales={"tn": tsc}))
    assert torch.equal(dest["plain"].cpu(), sd["plain"]) and torch.equal(dest["byte"].cpu(), sd["byte"])
    want_q, want_s = block_quantize(sd["blk"].float().numpy())
    assert np.array_equal(dest["blk"].view(torch.uint8).cpu().numpy(), want_q)
    assert np.array_equal(bs.cpu().numpy().view(np.uint32), want_s.view(np.uint32))
    assert_oracle(dest["ch"], cs, sd["ch"].float().numpy(), "channel")
    assert_oracle(dest["tn"], tsc, sd["tn"].float().numpy(), "tensor")
    assert sync._block_plans and sync._scaled_plans and set(sync.last_pull_ms) == {0} and sync.last_pull_ms[0] > 0
    with pytest.raises(ValueError, match="'ch'"):  # one name, two scale layouts
        run(DirectWeightSyncDest().pull({k: [h] for k, h in handles.items()}, dest, channel_scales={"ch": cs},
                                        tensor_scales={"ch": tsc}))
    sync.close()
    run(src.cleanup())


def test_replay_refresh_and_invalidation():
    full = rand_full((300, 260), torch.bfloat16, 5)
    sources, handles = register_boxes(full, [shard_box(full.shape, 4, r, 0) for r in range(4)])
    dst = shard_box(full.shape, 2, 1, 1)
    sync, q, s, _ = pull_box(handles, full.shape, dst, E4M3, granularity="tensor")
    plan = sync._scaled_plans[0]
    dsl = TensorSlice(dst[0], (0,), tuple(full.shape), dst[1], (1,))
    dest, scales = {"w": q}, {"w": s}
    before = _native.launch_count()
    run(sync.pull({"w": handles}, dest, {"w": dsl}, tensor_scales=scales))
    run(sync.pull({"w": handles}, dest, {"w": dsl}, tensor_scales=scales))
    assert _native.launch_count() == before + 4 and sync._scaled_plans[0] == plan  # replayed: two passes each
    for _, shard, _ in sources:
        shard.mul_(-7.0)
    new_full = (full.to(DEV) * -7.0).to(torch.bfloat16).cpu()
    run(sync.pull({"w": handles}, dest, {"w": dsl}, tensor_scales=scales))  # amax words re-armed: a smaller amax is seen
    assert_oracle(q, s, region(new_full, *dst).float().numpy(), "tensor")
    for _, shard, _ in sources:
        shard.mul_(0.25)
    full = (new_full.to(DEV) * 0.25).to(torch.bfloat16).cpu()
    run(sync.pull({"w": handles}, dest, {"w": dsl}, tensor_scales=scales))  # a smaller amax than the last run's
    assert_oracle(q, s, region(full, *dst).float().numpy(), "tensor")
    s2 = torch.zeros_like(s)
    run(sync.pull({"w": handles}, dest, {"w": dsl}, tensor_scales={"w": s2}))
    assert sync._scaled_plans[0] != plan  # a new scale tensor: the plan is rebuilt for it
    assert torch.equal(s2.view(torch.int32), s.view(torch.int32))
    plan = sync._scaled_plans[0]
    q2 = torch.zeros_like(q)
    run(sync.pull({"w": handles}, {"w": q2}, {"w": dsl}, tensor_scales={"w": s2}))
    assert sync._scaled_plans[0] != plan and torch.equal(q2.view(torch.uint8), q.view(torch.uint8))  # a new destination
    cs = torch.zeros(dst[1][0], 1, device=DEV)
    run(sync.pull({"w": handles}, {"w": q2}, {"w": dsl}, channel_scales={"w": cs}))  # same name, new granularity
    assert_oracle(q2, cs, region(full, *dst).float().numpy(), "channel")
    run(sync.pull({"w": handles}, {"w": q2}, {"w": dsl}))  # scales dropped: plain e4m3 cast
    assert not sync._scaled_plans
    assert torch.equal(q2.view(torch.uint8), region(full, *dst).to(DEV).to(E4M3).view(torch.uint8))
    sync.close()
    cleanup(sources)


def test_put_and_get_state_dict_with_channel_and_tensor_scales():
    import torch.distributed as dist
    from torch.testing._internal.distributed.fake_pg import FakeStore

    async def main():
        dist.init_process_group("fake", store=FakeStore(), rank=0, world_size=1)
        await ts.initialize()
        try:
            src = {"a": torch.randn(256, 384, device=DEV).to(torch.bfloat16), "b": torch.randn(2, 64, 96, device=DEV).to(torch.bfloat16),
                   "norm": torch.randn(384, device=DEV).to(torch.bfloat16)}
            await ts.put_state_dict(src, "policy_sq", direct_rdma=True)
            dst = {"a": torch.zeros(256, 384, dtype=E4M3, device=DEV), "b": torch.zeros(2, 64, 96, dtype=E4M3, device=DEV),
                   "norm": torch.zeros(384, dtype=torch.bfloat16, device=DEV)}
            cs, tsc = {"a": torch.zeros(256, 1, device=DEV)}, {"b": torch.zeros(2, device=DEV)}
            for _ in range(2):
                out = await ts.get_state_dict("policy_sq", user_state_dict=dst, direct_rdma=True, channel_scales=cs,
                                              tensor_scales=tsc)
                assert out is dst
                assert_oracle(dst["a"], cs["a"], src["a"].float().cpu().numpy(), "channel")
                assert_oracle(dst["b"], tsc["b"], src["b"].float().cpu().numpy(), "tensor")
                assert torch.equal(dst["norm"], src["norm"])
                src["a"].mul_(0.5)
                src["b"].mul_(3.0)
                await ts.put_state_dict(None, "policy_sq", direct_rdma=True)
            for kw in ({"channel_scales": cs}, {"tensor_scales": tsc}):
                with pytest.raises(NotImplementedError):
                    await ts.get_state_dict("policy_sq", user_state_dict=dst, **kw)
        finally:
            await ts.shutdown()
            dist.destroy_process_group()

    run(main())


def test_every_validation_error_raises_before_any_launch():
    full = rand_full((300, 260), torch.bfloat16, 6)
    sources, handles = register_boxes(full, [shard_box(full.shape, 4, r, 0) for r in range(4)])
    fp8_sources, fp8_handles = register_boxes(full.to(E4M3), [((0, 0), (300, 260))])
    q = torch.zeros(300, 260, dtype=E4M3, device=DEV)
    c, t = torch.zeros(300, 1, device=DEV), torch.zeros((), device=DEV)
    cases = [
        (TypeError, {"w": handles}, {"w": torch.zeros(300, 260, dtype=torch.bfloat16, device=DEV)}, c, t),  # bf16 destination
        (TypeError, {"w": fp8_handles}, {"w": q}, c, t),  # fp8 handles
        (ValueError, {"w": handles}, {"w": q}, torch.zeros(300, device=DEV), torch.zeros(2, device=DEV)),  # wrong scale shapes
        (ValueError, {"w": handles}, {"w": q}, torch.zeros(1, 300, device=DEV), torch.zeros(1, 1, device=DEV)),
        (TypeError, {"w": handles}, {"w": q}, c.double(), t.double()),
        (TypeError, {"w": handles}, {"w": q}, [1.0] * 300, 1.0),  # not tensors
        (ValueError, {"w": handles}, {"w": q}, c.cpu(), t.cpu()),  # scale on the host
        (ValueError, {"w": handles}, {"w": q}, torch.zeros(300, 2, device=DEV)[:, :1], None),  # non-contiguous scale
        (ValueError, {"w": handles}, {"w": torch.zeros(260, 300, dtype=E4M3, device=DEV).t()}, c, t),
        (ValueError, {"w": handles}, {"w": torch.zeros(300 * 260, dtype=E4M3, device=DEV)}, torch.zeros(1, device=DEV), t),
        (ValueError, {"w": handles[:3]}, {"w": q}, c, t),  # rows 225.. uncovered
        (ValueError, {}, {"w": q}, c, t),  # no handles at all
    ]
    before = _native.launch_count()
    for i, (exc, h, dest, cscale, tscale) in enumerate(cases):
        for kw, scale in (("channel_scales", cscale), ("tensor_scales", tscale)):
            if scale is None:
                continue
            sync = DirectWeightSyncDest()
            with pytest.raises(exc) as e:
                run(sync.pull(h, dest, **{kw: {"w": scale}}))
            assert "'w'" in str(e.value), (i, kw, e.value)
            assert _native.launch_count() == before, (i, kw)
            assert not sync._scaled_plans and not sync._native_plans
            sync.close()
    for kw in ("channel_scales", "tensor_scales"):  # not a destination name
        with pytest.raises(ValueError, match=kw):
            run(DirectWeightSyncDest().pull({"w": handles}, {"w": q}, **{kw: {"v": c}}))
    with pytest.raises(ValueError, match="block_scales"):  # one name in two dicts
        run(DirectWeightSyncDest().pull({"w": handles}, {"w": q}, block_scales={"w": torch.zeros(3, 3, device=DEV)},
                                        tensor_scales={"w": t}))
    assert _native.launch_count() == before
    cleanup(sources)
    cleanup(fp8_sources)


@needs_two_gpus
@pytest.mark.parametrize("g", GRANULARITIES)
def test_pieces_read_over_peer_mappings(g):
    full = rand_full((300, 520), torch.bfloat16, 8)
    boxes = [shard_box(full.shape, 4, r, 0) for r in range(4)]
    sources, handles = [], []
    for r, b in enumerate(boxes):  # shards alternate between cuda:1 and cuda:0
        s_, h_ = register_boxes(full, [b], device=f"cuda:{1 - r % 2}")
        sources += s_
        handles += h_
    for d in range(2):
        dst = shard_box(full.shape, 2, d, 1)
        sync, q, s, (qb, sb) = pull_box(handles, full.shape, dst, E4M3, granularity=g)
        assert _native.plan_info(sync._scaled_plans[0]).remote_src_bytes > 0
        assert_oracle(q, s, region(full, *dst).float().numpy(), g)
        assert guards_intact(qb) and guards_intact(sb)
        sync.close()
    cleanup(sources)

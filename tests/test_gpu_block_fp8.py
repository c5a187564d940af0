"""Block-scaled FP8 pulls on the H100: bf16/f16/f32 handles quantised into float8_e4m3fn destinations
with one float32 scale_inv per 128x128 block, during the gather.  Checked bit for bit against the
numpy oracle (finite data) and against a torch-CUDA tensor/tensor rendering of the formula (special
values, NaN bytes included); reshards, mixed dicts, plan replay and invalidation, the public
state-dict API, validation before any launch, and peer-mapped sources on a second GPU."""

import numpy as np
import pytest
import torch

import torchstore_b200 as ts
from oracle.block_fp8_oracle import quantize
from tests.helpers import (DEV, E4M3, cleanup, guards_intact, native_session, needs_two_gpus, pull_box, rand_full, region,
                           register_boxes, run, shard_box)
from tests.quant_pull_regimes import assert_block_torch_cuda
from tests.test_block_fp8_cpu import fixture_cases
from torchstore_b200 import _native
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource
from torchstore_b200.transport.types import TensorSlice

pytestmark = pytest.mark.gpu
_init = pytest.fixture(scope="module", autouse=True)(native_session)


def assert_oracle(q, s, x_f32):
    want_q, want_s = quantize(x_f32)
    assert np.array_equal(q.view(torch.uint8).cpu().numpy(), want_q)
    assert np.array_equal(s.cpu().numpy().view(np.uint32), want_s.view(np.uint32))


FINITE = [c for c in fixture_cases() if "nonfinite" not in c[0]]


@pytest.mark.parametrize("case", FINITE, ids=lambda c: c[0])
def test_exact_match_pull_of_the_fixture_shapes(case):
    _, dtype, x, _, _ = case
    full = torch.from_numpy(x).to(getattr(torch, dtype))
    shape = tuple(full.shape)
    sources, handles = register_boxes(full, [((0,) * len(shape), shape)])
    sync, q, s, (qb, sb) = pull_box(handles, shape, ((0,) * len(shape), shape), E4M3, granularity="block")
    assert_oracle(q, s, x)
    assert guards_intact(qb) and guards_intact(sb)
    sync.close()
    cleanup(sources)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
def test_exact_match_pull_4096(dtype):
    full = rand_full((4096, 4096), dtype, 1)
    sources, handles = register_boxes(full, [((0, 0), (4096, 4096))])
    sync, q, s, (qb, sb) = pull_box(handles, full.shape, ((0, 0), (4096, 4096)), E4M3, granularity="block")
    assert_oracle(q, s, full.float().numpy())
    assert guards_intact(qb) and guards_intact(sb)
    assert sync._block_plans and _native.plan_info(sync._block_plans[0]).num_tiles == 32 * 32
    sync.close()
    cleanup(sources)


@pytest.mark.parametrize("case", [c for c in fixture_cases() if c[0].startswith(("nonfinite", "zeros", "huge"))],
                         ids=lambda c: c[0])
def test_special_value_blocks_match_torch_cuda_bit_for_bit(case):
    _, dtype, x, _, _ = case
    full = torch.from_numpy(x).to(getattr(torch, dtype))
    sources, handles = register_boxes(full, [((0, 0), tuple(full.shape))])
    sync, q, s, (qb, sb) = pull_box(handles, full.shape, ((0, 0), tuple(full.shape)), E4M3, granularity="block")
    assert_block_torch_cuda(q, s, full)
    assert guards_intact(qb) and guards_intact(sb)
    sync.close()
    cleanup(sources)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_fsdp_rows_of_75_to_tp_columns(dtype):
    full = rand_full((300, 520), dtype, 2)
    sources, handles = register_boxes(full, [shard_box(full.shape, 4, r, 0) for r in range(4)])
    for d in range(4):
        dst = shard_box(full.shape, 4, d, 1)
        sync, q, s, (qb, sb) = pull_box(handles, full.shape, dst, E4M3, granularity="block")
        assert_oracle(q, s, region(full, *dst).float().numpy())
        assert guards_intact(qb) and guards_intact(sb)
        sync.close()
    cleanup(sources)


def test_moe_stack_reshard():
    full = rand_full((3, 130, 260), torch.bfloat16, 3)
    sources, handles = register_boxes(full, [shard_box(full.shape, 3, r, 1) for r in range(3)])
    for d in range(2):
        dst = shard_box(full.shape, 2, d, 2)
        sync, q, s, _ = pull_box(handles, full.shape, dst, E4M3, granularity="block")
        assert_oracle(q, s, region(full, *dst).float().numpy())
        sync.close()
    cleanup(sources)


def test_mixed_dict_leaves_the_other_names_as_a_plain_pull():
    g = torch.Generator().manual_seed(4)
    sd = {"q": (torch.randn(300, 200, generator=g)).to(torch.bfloat16),
          "byte": torch.randn(96, 64, generator=g).to(torch.bfloat16),
          "cast": (torch.randn(128, 96, generator=g) * 100).to(torch.bfloat16)}
    src = DirectWeightSyncSource()
    handles = {k: [h] for k, h in src.register({k: v.to(DEV) for k, v in sd.items()}, rank=0).items()}

    def dests():
        return {"q": torch.zeros(300, 200, dtype=E4M3, device=DEV), "byte": torch.zeros(96, 64, dtype=torch.bfloat16, device=DEV),
                "cast": torch.zeros(128, 96, dtype=E4M3, device=DEV)}

    plain, mixed = dests(), dests()
    scale = torch.zeros(3, 2, device=DEV)
    a, b = DirectWeightSyncDest(), DirectWeightSyncDest()
    run(a.pull(handles, plain))
    before = _native.launch_count()
    run(b.pull(handles, mixed, block_scales={"q": scale}))
    assert _native.launch_count() == before + 2  # the byte/cast plan and the block-scaled plan
    assert torch.equal(mixed["byte"], plain["byte"])
    assert torch.equal(mixed["cast"].view(torch.uint8), plain["cast"].view(torch.uint8))
    assert_oracle(mixed["q"], scale, sd["q"].float().numpy())
    assert set(b.last_pull_ms) == {0} and b.last_pull_ms[0] > 0
    a.close()
    b.close()
    run(src.cleanup())


def test_replay_refresh_and_invalidation():
    full = rand_full((300, 260), torch.bfloat16, 5)
    sources, handles = register_boxes(full, [shard_box(full.shape, 4, r, 0) for r in range(4)])
    dst = shard_box(full.shape, 2, 1, 1)
    sync, q, s, _ = pull_box(handles, full.shape, dst, E4M3, granularity="block")
    plan = sync._block_plans[0]
    dsl = TensorSlice(dst[0], (0,), tuple(full.shape), dst[1], (1,))
    dest, scales = {"w": q}, {"w": s}
    before = _native.launch_count()
    run(sync.pull({"w": handles}, dest, {"w": dsl}, block_scales=scales))
    run(sync.pull({"w": handles}, dest, {"w": dsl}, block_scales=scales))
    assert _native.launch_count() == before + 2 and sync._block_plans[0] == plan  # replayed
    for _, shard, _ in sources:
        shard.mul_(-7.0)
    new_full = (full.to(DEV) * -7.0).to(torch.bfloat16).cpu()
    run(sync.pull({"w": handles}, dest, {"w": dsl}, block_scales=scales))
    assert_oracle(q, s, region(new_full, *dst).float().numpy())
    s2 = torch.zeros_like(s)
    run(sync.pull({"w": handles}, dest, {"w": dsl}, block_scales={"w": s2}))
    assert sync._block_plans[0] != plan  # a new scale tensor: the plan is rebuilt for it
    assert torch.equal(s2.view(torch.int32), s.view(torch.int32))
    run(sync.pull({"w": handles}, dest, {"w": dsl}))  # block_scales dropped: plain e4m3 cast
    assert not sync._block_plans
    assert torch.equal(q.view(torch.uint8), region(new_full, *dst).to(DEV).to(E4M3).view(torch.uint8))
    sync.close()
    cleanup(sources)


def test_put_and_get_state_dict_with_block_scales():
    import torch.distributed as dist
    from torch.testing._internal.distributed.fake_pg import FakeStore

    async def main():
        dist.init_process_group("fake", store=FakeStore(), rank=0, world_size=1)
        await ts.initialize()
        try:
            src = {"w": torch.randn(256, 384, device=DEV).to(torch.bfloat16), "norm": torch.randn(384, device=DEV).to(torch.bfloat16)}
            await ts.put_state_dict(src, "policy_bq", direct_rdma=True)
            dst = {"w": torch.zeros(256, 384, dtype=E4M3, device=DEV), "norm": torch.zeros(384, dtype=torch.bfloat16, device=DEV)}
            scales = {"w": torch.zeros(2, 3, device=DEV)}
            out = await ts.get_state_dict("policy_bq", user_state_dict=dst, direct_rdma=True, block_scales=scales)
            assert out is dst
            assert_oracle(dst["w"], scales["w"], src["w"].float().cpu().numpy())
            assert torch.equal(dst["norm"], src["norm"])
            src["w"].mul_(0.5)
            await ts.put_state_dict(None, "policy_bq", direct_rdma=True)
            await ts.get_state_dict("policy_bq", user_state_dict=dst, direct_rdma=True, block_scales=scales)
            assert_oracle(dst["w"], scales["w"], src["w"].float().cpu().numpy())
            with pytest.raises(NotImplementedError):
                await ts.get_state_dict("policy_bq", user_state_dict=dst, block_scales=scales)
        finally:
            await ts.shutdown()
            dist.destroy_process_group()

    run(main())


def test_every_validation_error_raises_before_any_launch():
    full = rand_full((300, 260), torch.bfloat16, 6)
    sources, handles = register_boxes(full, [shard_box(full.shape, 4, r, 0) for r in range(4)])
    fp8_sources, fp8_handles = register_boxes(full.to(E4M3), [((0, 0), (300, 260))])
    q = torch.zeros(300, 260, dtype=E4M3, device=DEV)
    s = torch.zeros(3, 3, device=DEV)
    cases = [
        (TypeError, {"w": handles}, {"w": torch.zeros(300, 260, dtype=torch.bfloat16, device=DEV)}, {"w": s}),  # bf16 destination
        (TypeError, {"w": fp8_handles}, {"w": q}, {"w": s}),  # fp8 handles
        (ValueError, {"w": handles}, {"w": q}, {"w": torch.zeros(3, 2, device=DEV)}),  # wrong scale shape
        (TypeError, {"w": handles}, {"w": q}, {"w": torch.zeros(3, 3, dtype=torch.float64, device=DEV)}),
        (ValueError, {"w": handles}, {"w": q}, {"w": torch.zeros(3, 3)}),  # scale on the host
        (ValueError, {"w": handles}, {"w": q}, {"w": torch.zeros(3, 6, device=DEV)[:, ::2]}),  # non-contiguous scale
        (ValueError, {"w": handles}, {"w": torch.zeros(260, 300, dtype=E4M3, device=DEV).t()}, {"w": s}),
        (ValueError, {"w": handles}, {"w": torch.zeros(300 * 260, dtype=E4M3, device=DEV)}, {"w": torch.zeros(1, device=DEV)}),
        (ValueError, {"w": handles[:3]}, {"w": q}, {"w": s}),  # rows 225.. uncovered
        (ValueError, {"w": handles}, {"w": q}, {"v": s}),  # not a destination name
        (ValueError, {}, {"w": q}, {"w": s}),  # no handles at all
    ]
    before = _native.launch_count()
    for i, (exc, h, dest, scales) in enumerate(cases):
        sync = DirectWeightSyncDest()
        with pytest.raises(exc) as e:
            run(sync.pull(h, dest, block_scales=scales))
        if i == 8:
            assert "'w'" in str(e.value)
        assert _native.launch_count() == before, i
        assert not sync._block_plans and not sync._native_plans
        sync.close()
    cleanup(sources)
    cleanup(fp8_sources)


@needs_two_gpus
def test_pieces_read_over_peer_mappings():
    full = rand_full((300, 520), torch.bfloat16, 8)
    boxes = [shard_box(full.shape, 4, r, 0) for r in range(4)]
    sources, handles = [], []
    for r, b in enumerate(boxes):  # shards alternate between cuda:1 and cuda:0
        s_, h_ = register_boxes(full, [b], device=f"cuda:{1 - r % 2}")
        sources += s_
        handles += h_
    for d in range(2):
        dst = shard_box(full.shape, 2, d, 1)
        sync, q, s, (qb, sb) = pull_box(handles, full.shape, dst, E4M3, granularity="block")
        assert _native.plan_info(sync._block_plans[0]).remote_src_bytes > 0
        assert_oracle(q, s, region(full, *dst).float().numpy())
        assert guards_intact(qb) and guards_intact(sb)
        sync.close()
    cleanup(sources)

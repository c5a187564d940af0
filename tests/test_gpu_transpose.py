"""Transposed packed parts on the GPU: a grouped-GEMM trainer's input-major MoE stacks (FSDP shards simulated on cuda:0)
pulled into vLLM's output-major w13_weight / w2_weight, and transposed boxes of every element size, fused cast,
alignment and layout.  Every result is compared bit for bit with ``src.transpose(-2, -1).to(dst)`` in torch or with
transpose_oracle (alone, or composed with packed_oracle)."""

import numpy as np
import pytest
import torch

import workloads
from oracle import transpose_oracle as to
from tests.helpers import (DEV, E4M3, as_np, fsdp_handles, masters, needs_two_gpus, nv_handles, pull, pull_args, region,
                           run, whole_handle)
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, NvlinkBuffer, PackedPart, RDMAWeightHandle
from torchstore_b200.transport.types import TensorSlice

pytestmark = pytest.mark.gpu
QWEN = workloads.QWEN3_MOE
E5M2 = torch.float8_e5m2


def i16(shape):
    return torch.full(shape, -3, dtype=torch.int16, device=DEV).view(torch.bfloat16)


def grouped(scale=16, n_experts=16):
    return workloads.qwen3_moe_layout(QWEN, n_layers=1, scale=scale, with_embeddings=False, n_experts=n_experts,
                                      grouped_experts=True)


def bits(t):
    return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


# -- grouped Qwen3-MoE -> vLLM ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("tp,ep,n", [(1, False, 1), (2, False, 3), (8, False, 1), (8, False, 3), (2, True, 1),
                                     (8, True, 3)])
def test_qwen3_grouped_to_vllm_every_rank(tp, ep, n):
    """Scaled-down Qwen3-MoE (dim 128, 16 experts of width 48), grouped FSDP(n) -> vLLM TP(tp) or EP, every rank and
    every parameter, against transpose_oracle.  FSDP(3)'s uneven shards cut the expert dim."""
    layout = grouped()
    full = masters(layout, tp * 10 + n + ep)
    handles = nv_handles(layout, n, full)
    np_full = {k: as_np(v) for k, v in full.items()}
    for rank in range(tp):
        vl = workloads.vllm_tp_layout(layout, QWEN, tp, rank, ep=ep)
        dests, slices, packed = pull_args(vl, tp, rank, lambda _, s: i16(s))
        assert all(p.transpose for k in packed if ".experts." in k for p in packed[k])
        sync = pull(handles, dests, slices, packed=packed)
        assert sync._transpose_plans
        for name, entry in vl.items():
            want = to.destination(entry, np_full, name, fill_value=-3, dtype=np.int16)
            assert np.array_equal(as_np(dests[name]), want), (rank, name)
        sync.close()


@pytest.mark.parametrize("tp,rank,ep", [(8, 3, False), (8, 6, True)])
def test_qwen3_30b_a3b_full_size_layer(tp, rank, ep):
    """One full-size Qwen3-30B-A3B layer's experts (128 x [2048, 768] for each of w1 / w3 / w2), FSDP(3) -> one TP8
    or EP8 rank, against ``src.transpose(-2, -1)`` in torch."""
    layout = {k: v for k, v in grouped(scale=1, n_experts=None).items() if ".experts.w" in k}
    full = masters(layout, 5)
    handles = nv_handles(layout, 3, full)
    vl = workloads.vllm_tp_layout({**layout, "model.layers.0.mlp.gate.weight": ((128, 2048), ("R",))}, QWEN, tp, rank,
                                  ep=ep)
    names = [k for k in vl if k.endswith(("w13_weight", "w2_weight"))]
    dests = {k: i16(vl[k][0]) for k in names}
    pull(handles, dests, packed={k: vl[k][1] for k in names}).close()
    ex = "model.layers.0.mlp.experts."
    e_r, f_r = (16, 768) if ep else (128, 96)
    e0, f0 = (rank * 16, 0) if ep else (0, rank * 96)
    w1, w3, w2 = (full[ex + w][e0:e0 + e_r] for w in ("w1", "w3", "w2"))
    want13 = torch.cat([w1[:, :, f0:f0 + f_r].transpose(-2, -1), w3[:, :, f0:f0 + f_r].transpose(-2, -1)], dim=1)
    assert torch.equal(bits(dests[ex + "w13_weight"]), bits(want13))
    assert torch.equal(bits(dests[ex + "w2_weight"]), bits(w2[:, f0:f0 + f_r, :].transpose(-2, -1)))


# -- element sizes, casts, alignment -----------------------------------------------------------------------------------
def one_part(src, dest, index, offsets, n=1, dim=0):
    shape = tuple(src.shape)
    handles = fsdp_handles({"s": (shape, None)}, n, lambda _, off, loc: NvlinkBuffer(region(src, off, loc).contiguous()))
    if dim:  # shards cut along another dim
        handles = {"s": []}
        for r in range(n):
            off, loc = workloads.shard_box(shape, n, r, ("S", dim))
            handles["s"].append(RDMAWeightHandle(NvlinkBuffer(region(src, off, loc).contiguous()),
                                                 TensorSlice(off, (r,), shape, loc, (n,)), r))
    part = PackedPart("s", index, offsets, transpose=True)
    return pull(handles, {"d": dest}, packed={"d": (part,)}), part


@pytest.mark.parametrize("dtype", [torch.uint8, torch.int16, torch.int32, torch.int64, torch.bfloat16, torch.float32])
def test_same_dtype_every_element_size(dtype):
    g = torch.Generator(DEV).manual_seed(dtype.itemsize)
    if dtype.is_floating_point:
        src = torch.randn(3, 130, 200, generator=g, device=DEV).to(dtype)
    else:
        src = torch.randint(0, 127, (3, 130, 200), generator=g, device=DEV, dtype=torch.int64).to(dtype)
    dest = torch.zeros(3, 200, 130, dtype=dtype, device=DEV)
    one_part(src, dest, (slice(0, 3), slice(0, 200), slice(0, 130)), (0, 0, 0))[0].close()
    assert torch.equal(bits(dest), bits(src.transpose(-2, -1)))


def special_values(dtype, shape, seed):
    """Random values with NaN, +-Inf, subnormals, zeros of both signs and fp8-overflowing magnitudes sprinkled in."""
    g = torch.Generator(DEV).manual_seed(seed)
    if dtype.itemsize == 1:  # every fp8 byte pattern, NaNs and (e5m2) Infs included
        return torch.randint(0, 256, shape, generator=g, device=DEV, dtype=torch.uint8).view(dtype)
    x = torch.randn(shape, generator=g, device=DEV, dtype=torch.float64) * 100
    specials = torch.tensor([float("nan"), float("inf"), -float("inf"), 0.0, -0.0, 1e-40, -3e-42, 6e-8, 1e-5, 448.0,
                             460.0, 465.0, -500.0, 57344.0, 61440.0, 70000.0, 1e30, 3.5e38, 1e300, 1e-310],
                            dtype=torch.float64, device=DEV)
    flat = x.view(-1)
    idx = torch.randint(0, flat.numel(), (flat.numel() // 7,), generator=g, device=DEV)
    flat[idx] = specials[torch.randint(0, specials.numel(), idx.shape, generator=g, device=DEV)]
    return x.to(dtype)


CASTS = [(a, b) for a in (torch.float32, torch.bfloat16, torch.float16) for b in (torch.float32, torch.bfloat16,
                                                                                   torch.float16, E4M3, E5M2) if a != b]
CASTS += [(a, b) for a in (E4M3, E5M2) for b in (torch.float32, torch.bfloat16, torch.float16)]
CASTS += [(torch.float64, torch.float32), (torch.float32, torch.float64)]


@pytest.mark.parametrize("sdt,ddt", CASTS, ids=[f"{a}-{b}".replace("torch.", "") for a, b in CASTS])
def test_every_fused_cast_bit_exact_with_torch(sdt, ddt):
    """Bit for bit with torch's .to(); an fp8 NaN widened into f32 is any NaN (as for the copy kernel's casts), and
    there the result is bit for bit the copy kernel's own cast of the transposed source."""
    src = special_values(sdt, (2, 67, 150), len(str(sdt)) + len(str(ddt)))
    dest = torch.zeros(2, 150, 67, dtype=ddt, device=DEV)
    one_part(src, dest, (slice(0, 2), slice(0, 150), slice(0, 67)), (0, 0, 0))[0].close()
    want = src.transpose(-2, -1).to(ddt)
    if sdt.itemsize == 1 and ddt == torch.float32:
        nan = torch.isnan(want)
        assert torch.equal(torch.isnan(dest), nan) and torch.equal(bits(dest)[~nan], bits(want)[~nan])
        copied = torch.zeros_like(dest)
        pull({"s": whole_handle(src.transpose(-2, -1).contiguous())}, {"s": copied}).close()
        assert torch.equal(bits(dest), bits(copied))
    else:
        assert torch.equal(bits(dest), bits(want))


@pytest.mark.parametrize("n,dim", [(1, 0), (3, 1), (3, 2)])
def test_unaligned_and_odd_boxes(n, dim):
    """A (5, 37, 51) box at odd offsets of a (5, 41, 60) destination, read at source (0, 2, 1): neither side's rows
    start 16-byte aligned, and no extent is a tile multiple."""
    g = torch.Generator(DEV).manual_seed(n + dim)
    src = (torch.randn(5, 53, 40, generator=g, device=DEV)).to(torch.bfloat16)
    dest = i16((5, 41, 60))
    index = (slice(0, 5), slice(3, 40), slice(1, 52))
    sync, part = one_part(src, dest, index, (0, 2, 1), n, dim)
    sync.close()
    want = to.fill(np.full((5, 41, 60), -3, dtype=np.int16), [part], {"s": as_np(src)})
    assert np.array_equal(as_np(dest), want)


def test_mixed_transposed_and_untransposed_parts():
    g = torch.Generator(DEV).manual_seed(3)
    w = torch.randn(4, 24, 8, generator=g, device=DEV).to(torch.bfloat16)
    v = torch.randn(4, 8, 24, generator=g, device=DEV).to(torch.bfloat16)
    u = torch.randn(30, 9, generator=g, device=DEV).to(torch.bfloat16)
    parts = (PackedPart("w", (slice(0, 4), slice(0, 8), slice(0, 24)), (0, 0, 0), transpose=True),
             PackedPart("v", (slice(0, 4), slice(8, 16), slice(0, 24)), (0, 0, 0)),
             PackedPart("u", (1, slice(16, 20), slice(0, 24)), (3, 5), transpose=True))
    dest = i16((4, 20, 24))
    sync = pull({"w": whole_handle(w), "v": whole_handle(v), "u": whole_handle(u)}, {"d": dest}, packed={"d": parts})
    assert sync._transpose_plans and sync.plan_info()[0]["num_rects"] == 1
    sync.close()
    want = to.fill(np.full((4, 20, 24), -3, dtype=np.int16), parts, {"w": as_np(w), "v": as_np(v), "u": as_np(u)})
    assert np.array_equal(as_np(dest), want)


def test_plan_reuse_and_rebuild_when_transpose_flips():
    g = torch.Generator(DEV).manual_seed(4)
    src = torch.randn(2, 32, 32, generator=g, device=DEV).to(torch.bfloat16)
    handles = {"s": whole_handle(src)}
    dest = i16((2, 32, 32))
    dests = {"d": dest}
    packed = {"d": (PackedPart("s", (slice(0, 2), slice(0, 32), slice(0, 32)), (0, 0, 0), transpose=True),)}
    sync = DirectWeightSyncDest()
    run(sync.pull(handles, dests, packed=packed))
    plan = sync._plan
    run(sync.pull(handles, dests, packed=packed))
    assert sync._plan is plan and sync.last_pull_ms[0] > 0
    want = to.fill(np.zeros((2, 32, 32), dtype=np.int16), packed["d"], {"s": as_np(src)})
    assert np.array_equal(as_np(dest), want)
    flipped = {"d": (PackedPart("s", (slice(0, 2), slice(0, 32), slice(0, 32)), (0, 0, 0), transpose=False),)}
    run(sync.pull(handles, dests, packed=flipped))
    assert sync._plan is not plan and not sync._transpose_plans
    assert torch.equal(bits(dest), bits(src))
    run(sync.pull(handles, dests, packed=packed))
    assert sync._transpose_plans and np.array_equal(as_np(dest), want)
    sync.close()


def test_scaled_destination_is_refused_before_compiling():
    src = torch.randn(16, 8, device=DEV).to(torch.bfloat16)
    dest = torch.zeros(8, 16, dtype=E4M3, device=DEV)
    packed = {"d": (PackedPart("s", (slice(0, 8), slice(0, 16)), (0, 0), transpose=True),)}
    with pytest.raises(ValueError, match=r"packed destination 'd' part 0 \(source 's'\): a transposed part takes "
                                         r"element-wise routes only .* channel_scales"):
        pull({"s": whole_handle(src)}, {"d": dest}, packed=packed, channel_scales={"d": torch.zeros(8, 1, device=DEV)})


# -- the public path ----------------------------------------------------------------------------------------------------
def test_get_state_dict_with_transposed_parts():
    import torch.distributed as dist
    from torch.testing._internal.distributed.fake_pg import FakeStore

    import torchstore_b200 as ts

    layout = {k: v for k, v in grouped().items() if ".experts.w" in k}
    full = masters(layout, 71)
    vl = workloads.vllm_tp_layout({**layout, "model.layers.0.mlp.gate.weight": ((16, 128), ("R",))}, QWEN, 2, 1)
    packed = {n: parts for n, (_, parts, _) in vl.items() if parts}

    async def main():
        dist.init_process_group("fake", store=FakeStore(), rank=0, world_size=1)
        await ts.initialize()
        try:
            await ts.put_state_dict(full, "policy_grouped", direct_rdma=True)
            dst = {n: torch.zeros(vl[n][0], dtype=torch.bfloat16, device=DEV) for n in packed}
            for _ in range(2):
                out = await ts.get_state_dict("policy_grouped", user_state_dict=dst, direct_rdma=True, packed=packed)
                assert out is dst
                np_full = {k: as_np(v) for k, v in full.items()}
                for n in packed:
                    want = to.destination(vl[n], np_full, n, dtype=np.int16)
                    assert np.array_equal(as_np(dst[n]), want), n
                for t in full.values():
                    t.mul_(2)
        finally:
            await ts.shutdown()
            dist.destroy_process_group()

    run(main())


@needs_two_gpus
def test_transposed_parts_read_over_peer_mappings():
    layout = grouped(scale=8)
    full = masters(layout, 81, device="cuda:1")
    handles = nv_handles(layout, 2, full)
    vl = workloads.vllm_tp_layout(layout, QWEN, 2, 0)
    dests, slices, packed = pull_args(vl, 2, 0, lambda _, s: i16(s))
    pull(handles, dests, slices, packed=packed).close()
    np_full = {k: as_np(v) for k, v in full.items()}
    for name, entry in vl.items():
        assert np.array_equal(as_np(dests[name]), to.destination(entry, np_full, name, fill_value=-3, dtype=np.int16)), name

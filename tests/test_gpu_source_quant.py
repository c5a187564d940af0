"""Source-side quantisation on the H100: DirectWeightSyncSource.register(quantize=...) staging bit for bit against
the numpy oracle (finite groups) and torch CUDA (NaN bytes included), full-tensor equivalence at group-aligned
shard boundaries, refresh replay, guard bytes around the kernel's outputs, the three existing consumers of scaled
handles, mixed registers and the state-dict API.  Several "ranks" are emulated as several sources on cuda:0."""

import numpy as np
import pytest
import torch

import torchstore_b200 as ts
from oracle import block_fp8_oracle
from oracle.source_quant_oracle import GRANULARITIES, element_scales, synth_f32, torch_quantize
from tests.helpers import DEV, E4M3, cleanup, needs_two_gpus, register_boxes, run
from tests.source_quant_regimes import assert_exact
from tests.test_source_quant_cpu import CODE, DT
from torchstore_b200 import _native
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource, ScaledNvlinkBuffer
from torchstore_b200.launch import Plans
from torchstore_b200.transport.types import TensorSlice

pytestmark = pytest.mark.gpu
DTYPES = (torch.bfloat16, torch.float16, torch.float32)


def row_bounds(n: int, k: int) -> list[tuple[int, int]]:
    """FSDP row split of n rows over k ranks (the first ranks take one more row when k does not divide n)."""
    step, extra = divmod(n, k)
    out, r = [], 0
    for i in range(k):
        e = r + step + (1 if i < extra else 0)
        out.append((r, e))
        r = e
    return out


def row_boxes(shape, bounds, cols=None):
    """(offsets, local shape) of each row range of `bounds` (within the column range `cols`, all columns without)."""
    c0, c1 = cols or (0, shape[-1])
    lead = tuple(shape[:-2])
    return [((0,) * len(lead) + (r0, c0), lead + (r1 - r0, c1 - c0)) for r0, r1 in bounds]


def staging(src: DirectWeightSyncSource, name="w"):
    q, s, _ = src._quantized[name]
    return q, s


LAYOUTS = {"aligned_4x128": ((512, 384), row_bounds(512, 4), None),
           "uneven_300_over_4": ((300, 520), row_bounds(300, 4), None),
           "col_shard_at_70": ((256, 300), row_bounds(256, 2), (70, 262))}


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("g", GRANULARITIES)
def test_staging_is_exact(g, dtype, layout):
    shape, bounds, cols = LAYOUTS[layout]
    full = synth_f32(shape, 11 + len(bounds)).to(dtype)
    full[bounds[-1][0] + 3, 5] = float("nan")  # a NaN group in the last shard
    sources, handles = register_boxes(full, row_boxes(full.shape, bounds, cols), quantize={"w": g})
    c0 = cols[0] if cols else 0
    for (src, shard, _), (r0, _), h in zip(sources, bounds, handles):
        q, s = staging(src)
        assert isinstance(h.rdma_buffer, ScaledNvlinkBuffer) and (h.rdma_buffer.row0, h.rdma_buffer.col0) == (r0, c0)
        assert h.rdma_buffer.granularity == g and h.rdma_buffer.dtype == E4M3
        assert_exact(q, s, shard, g, r0, c0)
    cleanup(sources)


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
def test_moe_stack_and_long_rows(dtype):
    x = synth_f32((3, 130, 260), 21).to(dtype)
    for g in GRANULARITIES:
        sources, _ = register_boxes(x, row_boxes(x.shape, [(0, 130)]), quantize={"w": g})
        q, s = staging(sources[0][0])
        assert_exact(q, s, sources[0][1], g, 0, 0)
        cleanup(sources)
    long = synth_f32((4, 16400 if dtype != torch.float32 else 8200), 22).to(dtype)  # rows over the 32 KiB stage
    long[2, 7] = float("inf")
    sources, _ = register_boxes(long, row_boxes(long.shape, [(0, 4)]), quantize={"w": "channel"})
    q, s = staging(sources[0][0])
    assert_exact(q, s, sources[0][1], "channel", 0, 0)
    cleanup(sources)


@pytest.mark.parametrize("g", ("block", "channel"))
def test_group_aligned_shards_equal_the_full_tensor(g):
    full = synth_f32((1024, 640), 31).to(torch.bfloat16)
    sources, _ = register_boxes(full, row_boxes(full.shape, row_bounds(1024, 8)), quantize={"w": g})
    q = torch.cat([staging(src)[0].view(torch.uint8) for src, *_ in sources])
    s = torch.cat([staging(src)[1] for src, *_ in sources])
    fq, fs = torch_quantize(full.to(DEV), g)
    assert torch.equal(q, fq.view(torch.uint8)) and torch.equal(s.view(torch.int32), fs.view(torch.int32))
    cleanup(sources)


@pytest.mark.parametrize("g", GRANULARITIES)
def test_refresh_after_an_in_place_update(g):
    full = synth_f32((300, 520), 41).to(torch.bfloat16)
    sources, _ = register_boxes(full, row_boxes(full.shape, row_bounds(300, 3)), quantize={"w": g})
    for step in range(2):
        for src, shard, _ in sources:
            shard.mul_(0.25)
            before = staging(src)[1].clone()
            assert src.refresh() == 1
            q, s = staging(src)
            assert_exact(q, s, shard, g, src._handles["w"].rdma_buffer.row0, 0)
            if g == "tensor":  # smaller values, smaller scale: the amax words start from zero on every replay
                assert float(s) < float(before)
    cleanup(sources)


@pytest.mark.parametrize("g", GRANULARITIES)
@pytest.mark.parametrize("misalign", (0, 1))
def test_kernel_writes_nothing_outside_its_outputs(g, misalign):
    """The plan driven directly on guarded buffers: bytes around the fp8 output and the scale stay intact, with an
    unaligned shard offset and (misalign=1) a source address that is not 16-byte aligned."""
    shape, r0, c0 = (3, 130, 260), 37, 70
    x = synth_f32(shape, 51).to(torch.bfloat16)
    flat = torch.zeros(x.numel() + 64, dtype=torch.bfloat16, device=DEV)
    src = flat[misalign: misalign + x.numel()].view(shape)
    src.copy_(x.to(DEV))
    from torchstore_b200.direct_weight_sync import source_scale_shapes

    sshape = source_scale_shapes(g, shape, r0, c0)[0]
    n_s = int(np.prod(sshape)) if sshape else 1
    qbuf = torch.full((x.numel() + 512,), 0xAB, dtype=torch.uint8, device=DEV)
    sbuf = torch.full((n_s + 128,), -7.0, device=DEV)
    q, s = qbuf[256: 256 + x.numel()], sbuf[64: 64 + n_s]
    t = _native.SourceQuantTarget(src.data_ptr(), q.data_ptr(), s.data_ptr(), 3, 130, 260, r0, c0, DT["bfloat16"], CODE[g])
    plans = Plans.build_source_quant({0: [t]})
    try:
        for _ in range(2):
            plans.launch()
            plans.synchronize()
    finally:
        plans.close()
    assert_exact(q.view(E4M3).view(shape), s.view(sshape), x, g, r0, c0)
    assert (qbuf[:256] == 0xAB).all() and (qbuf[256 + x.numel():] == 0xAB).all()
    assert (sbuf[:64] == -7.0).all() and (sbuf[64 + n_s:] == -7.0).all()


def assemble(sources, shape, bounds):
    """The published fp8 bytes and per-element f32 scales of all shards, assembled into the full tensor."""
    q = torch.zeros(shape, dtype=torch.uint8)
    es = torch.zeros(shape, dtype=torch.float32)
    for (src, *_), (r0, r1) in zip(sources, bounds):
        sq, ss = staging(src)
        g = src._handles["w"].rdma_buffer.granularity
        q[r0:r1] = sq.view(torch.uint8).cpu()
        es[r0:r1] = torch.from_numpy(np.ascontiguousarray(element_scales(ss.cpu().numpy(), g, sq.shape, r0, 0)))
    return q, es


@pytest.mark.parametrize("g", GRANULARITIES)
def test_consumers_dequantise_requantise_and_raw_bytes(g):
    shape, bounds = (300, 520), row_bounds(300, 4)
    full = synth_f32(shape, 61).to(torch.bfloat16)
    sources, handles = register_boxes(full, row_boxes(full.shape, bounds), quantize={"w": g})
    q, es = assemble(sources, shape, bounds)
    x32 = q.view(E4M3).float() * es  # what a dequantising pull into f32 writes
    for d in range(2):  # a TP(2) column split
        c0, c1 = d * 260, (d + 1) * 260
        tslice = TensorSlice((0, c0), (d,), shape, (300, 260), (2,))
        y = torch.zeros(300, 260, dtype=torch.bfloat16, device=DEV)
        sync = DirectWeightSyncDest()
        run(sync.pull({"w": handles}, {"w": y}, {"w": tslice}))
        assert torch.equal(y.cpu(), x32[:, c0:c1].to(torch.bfloat16))
        sync.close()
    # requantise into a full-size block-scaled destination
    yq = torch.zeros(shape, dtype=E4M3, device=DEV)
    ys = torch.zeros(3, 5, device=DEV)
    sync = DirectWeightSyncDest()
    run(sync.pull({"w": handles}, {"w": yq}, block_scales={"w": ys}, requantize=True))
    want_q, want_s = block_fp8_oracle.quantize(x32.numpy())
    assert np.array_equal(yq.view(torch.uint8).cpu().numpy(), want_q)
    assert np.array_equal(ys.cpu().numpy().view(np.uint32), want_s.view(np.uint32))
    sync.close()
    # an unscaled fp8 destination gets the staging bytes
    raw = torch.zeros(shape, dtype=E4M3, device=DEV)
    sync = DirectWeightSyncDest()
    run(sync.pull({"w": handles}, {"w": raw}))
    assert torch.equal(raw.view(torch.uint8).cpu(), q)
    sync.close()
    cleanup(sources)


def test_mixed_register():
    w = synth_f32((256, 384), 71).to(DEV)  # an fp32 master weight
    norm = synth_f32((1, 384), 72).reshape(384).to(DEV)
    src = DirectWeightSyncSource()
    h = src.register({"w": w, "norm": norm}, rank=0, transfer_dtype=torch.bfloat16, quantize={"w": "block"})
    assert h["w"].rdma_buffer.dtype == E4M3 and h["norm"].rdma_buffer.dtype == torch.bfloat16
    assert src.refresh() == 2
    assert_exact(*staging(src), w, "block", 0, 0)
    y = torch.zeros(384, dtype=torch.bfloat16, device=DEV)
    run(DirectWeightSyncDest().pull({"norm": [h["norm"]]}, {"norm": y}))
    assert torch.equal(y, norm.to(torch.bfloat16))
    run(src.cleanup())
    # beside a pre-scaled fp8 weight published with its scale
    fq, fs = torch_quantize(w, "channel")
    src = DirectWeightSyncSource()
    h = src.register({"w": w.to(torch.bfloat16), "f": fq}, rank=0, quantize={"w": "tensor"}, channel_scales={"f": fs})
    assert h["f"].rdma_buffer.granularity == "channel" and h["w"].rdma_buffer.granularity == "tensor"
    assert src.refresh() == 1
    assert_exact(*staging(src), w.to(torch.bfloat16), "tensor", 0, 0)
    y = torch.zeros(256, 384, device=DEV)
    run(DirectWeightSyncDest().pull({"f": [h["f"]]}, {"f": y}))
    assert torch.equal(y, fq.float() * fs)
    run(src.cleanup())


@pytest.mark.parametrize("rank", (0, 1, 3))
def test_dtensor_shard_takes_its_offset_from_the_dtensor(rank):
    """A row-sharded DTensor (300 rows over 4 ranks: torch puts rank r at row 75 r, mid-block) registered with quantize:
    the handle's (row0, col0) and the staging's groups come from the DTensor's layout."""
    import torch.distributed as dist
    from torch.distributed.device_mesh import DeviceMesh
    from torch.distributed.tensor import DTensor, Shard
    from torch.testing._internal.distributed.fake_pg import FakeStore

    full = synth_f32((300, 520), 101).to(torch.bfloat16)
    dist.init_process_group("fake", store=FakeStore(), rank=rank, world_size=4)
    try:
        mesh = DeviceMesh("cuda", torch.arange(4), _init_backend=False, _rank=rank)
        local = full[75 * rank: 75 * (rank + 1)].contiguous().to(DEV)
        dt = DTensor.from_local(local, mesh, (Shard(0),), run_check=False, shape=full.shape, stride=full.stride())
        for g in GRANULARITIES:
            src = DirectWeightSyncSource()
            h = src.register({"w": dt}, rank=rank, quantize={"w": g})["w"]
            assert (h.rdma_buffer.row0, h.rdma_buffer.col0) == (75 * rank, 0)
            assert tuple(h.tensor_slice.offsets) == (75 * rank, 0)
            assert_exact(*staging(src), local, g, 75 * rank, 0)
            run(src.cleanup())
    finally:
        dist.destroy_process_group()


def test_put_and_get_state_dict_with_quantize():
    import torch.distributed as dist
    from torch.testing._internal.distributed.fake_pg import FakeStore

    async def main():
        dist.init_process_group("fake", store=FakeStore(), rank=0, world_size=1)
        await ts.initialize()
        try:
            w = synth_f32((256, 384), 81).to(torch.bfloat16).to(DEV)
            src = {"w": w, "norm": torch.randn(384, device=DEV).to(torch.bfloat16)}
            await ts.put_state_dict(src, "policy_sq", direct_rdma=True, quantize={"w": "block"})
            dst = {"w": torch.zeros(256, 384, dtype=torch.bfloat16, device=DEV),
                   "norm": torch.zeros(384, dtype=torch.bfloat16, device=DEV)}
            for _ in range(2):
                out = await ts.get_state_dict("policy_sq", user_state_dict=dst, direct_rdma=True)
                assert out is dst
                q, s = torch_quantize(w, "block")
                es = s.repeat_interleave(128, 0).repeat_interleave(128, 1)[:256, :384]
                assert torch.equal(dst["w"], (q.float() * es).to(torch.bfloat16))
                assert torch.equal(dst["norm"], src["norm"])
                w.mul_(0.5)
                await ts.put_state_dict(None, "policy_sq", direct_rdma=True)
            with pytest.raises(NotImplementedError):
                await ts.put_state_dict(src, "policy_sq2", quantize={"w": "block"})
        finally:
            await ts.shutdown()
            dist.destroy_process_group()

    run(main())


@needs_two_gpus
@pytest.mark.parametrize("g", GRANULARITIES)
def test_quantised_handles_read_over_peer_mappings(g):
    shape, bounds = (300, 520), row_bounds(300, 2)
    full = synth_f32(shape, 91).to(torch.bfloat16)
    sources, handles = register_boxes(full, row_boxes(full.shape, bounds), device="cuda:1", quantize={"w": g})
    q, es = assemble(sources, shape, bounds)
    y = torch.zeros(shape, dtype=torch.bfloat16, device=DEV)
    sync = DirectWeightSyncDest()
    run(sync.pull({"w": handles}, {"w": y}))
    assert torch.equal(y.cpu(), (q.view(E4M3).float() * es).to(torch.bfloat16))
    sync.close()
    cleanup(sources)

"""Multi-GPU paths: P2P between two devices of one process, CUDA-IPC between two processes, and a
2-rank SPMD store with direct weight sync.  Skipped on boxes with a single GPU."""

import asyncio
import math
import os
import socket
import tempfile

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from tests.helpers import run

pytestmark = pytest.mark.gpu


def _ngpu():
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


needs2 = pytest.mark.skipif(_ngpu() < 2, reason="needs 2 GPUs")


@needs2
def test_p2p_pull_between_two_devices_single_process():
    from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource

    src = torch.arange(1 << 22, dtype=torch.int32, device="cuda:0").reshape(2048, 2048)
    handles = DirectWeightSyncSource().register({"w": src}, rank=0)
    dst = torch.zeros(2048, 2048, dtype=torch.int32, device="cuda:1")
    sync = DirectWeightSyncDest()
    run(sync.pull({"w": [handles["w"]]}, {"w": dst}))
    assert torch.equal(dst.cpu(), src.cpu())
    info = sync.plan_info()[1]
    assert info["remote_src_bytes"] == src.numel() * 4


@needs2
def test_store_get_across_devices_single_process(monkeypatch):
    import torchstore_b200 as ts

    async def main():
        await ts.initialize(num_storage_volumes=2, strategy=ts.LocalRankStrategy())
        try:
            monkeypatch.delenv("RANK", raising=False)
            monkeypatch.setenv("LOCAL_RANK", "1")
            t = torch.randn(1024, 512, device="cuda:1")
            await ts.put("t", t)  # lands in volume 1 = HBM of GPU 1
            monkeypatch.setenv("LOCAL_RANK", "0")
            dest = torch.zeros(1024, 512, device="cuda:0")
            await ts.get("t", dest)  # GPU 0 pulls over NVLink
            assert torch.equal(dest.cpu(), t.cpu())
        finally:
            await ts.shutdown()

    run(main())


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _free_ports(n):
    """n distinct free ports (all sockets held open until every port is chosen)."""
    socks = []
    for _ in range(n):
        s = socket.socket()
        s.bind(("127.0.0.1", 0))
        socks.append(s)
    ports = [s.getsockname()[1] for s in socks]
    for s in socks:
        s.close()
    return ports


def _ipc_worker(rank, world, port, pg_port, outdir, same_gpu):
    os.environ.update({"RANK": str(rank), "LOCAL_RANK": str(0 if same_gpu else rank), "WORLD_SIZE": str(world),
                       "LOCAL_WORLD_SIZE": str(world), "MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port)})
    os.environ.pop("TORCHELASTIC_USE_AGENT_STORE", None)
    import torch.distributed as dist

    import torchstore_b200 as ts

    dev = torch.device("cuda", 0 if same_gpu else rank)
    torch.cuda.set_device(dev)

    async def main():
        dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{pg_port}", rank=rank, world_size=world)
        await ts.initialize_spmd(ts.LocalRankStrategy())
        # every rank owns rows [rank*R, (rank+1)*R) of a [world*R, C] weight (FSDP Shard(0)) and
        # wants columns [rank*C/world, ...) of all rows (TP Shard(1))
        R, C = 256, 512
        full = torch.arange(world * R * C, dtype=torch.float32).reshape(world * R, C)
        mine = full[rank * R:(rank + 1) * R].contiguous().to(dev)
        from torchstore_b200.transport.types import TensorSlice

        src_slice = TensorSlice((rank * R, 0), (rank,), (world * R, C), (R, C), (world,))
        from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource

        source = DirectWeightSyncSource()
        handles = source.register({"w": mine}, rank=rank, tensor_slices={"w": src_slice})
        await ts.put(f"sync/rank_{rank}", handles)
        dist.barrier()
        all_handles = {"w": []}
        for r in range(world):
            all_handles["w"].append((await ts.get(f"sync/rank_{r}"))["w"])
        cw = C // world
        dest = torch.zeros(world * R, cw, device=dev)
        dslice = TensorSlice((0, rank * cw), (rank,), (world * R, C), (world * R, cw), (world,))
        sync = DirectWeightSyncDest()
        await sync.pull(all_handles, {"w": dest}, {"w": dslice})
        ok1 = torch.equal(dest.cpu(), full[:, rank * cw:(rank + 1) * cw])
        # second round after an in-place update on every source
        dist.barrier()
        mine.mul_(-1.0)
        torch.cuda.synchronize()
        dist.barrier()
        await sync.pull(all_handles, {"w": dest}, {"w": dslice})
        ok2 = torch.equal(dest.cpu(), -full[:, rank * cw:(rank + 1) * cw])
        # store path across processes: tensor put by rank r, read in place by the other rank
        await ts.put(f"t_{rank}", torch.full((128, 64), float(rank + 1), device=dev))
        dist.barrier()
        other = (rank + 1) % world
        got = await ts.get(f"t_{other}", torch.zeros(128, 64, device=dev))
        ok3 = bool((got == float(other + 1)).all().item())
        info = sync.plan_info()[dev.index]
        dist.barrier()
        sync.close()
        await ts.shutdown()
        dist.destroy_process_group()
        np.save(os.path.join(outdir, f"{rank}.npy"), np.array([ok1, ok2, ok3, info["remote_src_bytes"] > 0 or same_gpu]))

    asyncio.run(main())


@pytest.mark.parametrize("same_gpu", [True, False])
def test_two_process_ipc_direct_sync_and_store(same_gpu):
    """Cross-process handles: cudaIpc mapping of torch-allocated params (base handle + offset)."""
    if not same_gpu and _ngpu() < 2:
        pytest.skip("needs 2 GPUs")
    world = 2
    port, pg_port = _free_ports(2)
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_ipc_worker, args=(world, port, pg_port, d, same_gpu), nprocs=world, join=True)
        for r in range(world):
            assert np.load(os.path.join(d, f"{r}.npy")).all(), (r, np.load(os.path.join(d, f"{r}.npy")))


@needs2
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.int32])
def test_config2_flat_4gib_between_two_gpus(dtype):
    """BASELINE config #2: direct_weight_sync of a 4 GiB flat tensor GPU0 -> GPU1, same placement
    (one exact-match op); bf16 random weights and the int32 arange variant, bit-exact."""
    from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource

    nbytes = 4 << 30
    n = nbytes // dtype.itemsize
    if dtype == torch.int32:
        src = torch.arange(n, dtype=torch.int32, device="cuda:0")
    else:
        src = torch.empty(n, dtype=dtype, device="cuda:0").normal_(0, 0.02)
    handles = DirectWeightSyncSource().register({"flat": src}, rank=0)
    dst = torch.zeros(n, dtype=dtype, device="cuda:1")
    sync = DirectWeightSyncDest()
    run(sync.pull({"flat": [handles["flat"]]}, {"flat": dst}))
    assert len(sync._plan) == 1 and sync._plan[0].dest_tensor is None
    a = src.view(torch.int32) if dtype == torch.int32 else src.view(torch.int16)
    b = dst.view(torch.int32) if dtype == torch.int32 else dst.view(torch.int16)
    assert torch.equal(a.to("cuda:1"), b)  # bit-exact and order-sensitive at full size
    gbps = nbytes / sync.last_pull_ms[1] / 1e6
    print(f"config2 {dtype}: {sync.last_pull_ms[1]:.3f} ms, {gbps:.1f} GB/s")
    sync.close()


def _stale_exporter(conn):
    """Exports an allocation, frees it, allocates again (normally at the same address) and exports that."""
    from torchstore_b200 import _native

    _native.init()
    torch.cuda.set_device(0)
    size = 64 << 20
    for pattern in (1, 2):
        arena = _native.arena_create(0, size)
        ptr = _native.arena_alloc(arena, size)
        host = np.full(size, pattern, dtype=np.uint8)
        _native.memcpy_async(0, ptr, host.ctypes.data, size, _native.TSB_H2D)
        _native.stream_sync(0, None)
        conn.send(_native.region_to_bytes(_native.export_region(ptr, size)))
        assert conn.recv() == "done"
        _native.arena_destroy(arena)  # cudaFree: the importer's mapping now pins dead memory
    conn.close()


def test_importer_evicts_stale_mapping_when_exporter_reuses_the_address():
    """f3: a freed-and-reallocated exporter allocation gets a new IPC handle and a new epoch; the
    importer must map the new one and drop the mapping of the old one instead of keeping both
    (reference semantics: registration caches evict with the memory, torchcomms/cache.py:150-186)."""
    from torchstore_b200 import _native
    from torchstore_b200.planner import StridedMem, build_rects

    _native.init()
    ctx = mp.get_context("spawn")
    parent, child = ctx.Pipe()
    proc = ctx.Process(target=_stale_exporter, args=(child,))
    proc.start()
    before = _native.import_stats()
    regions = []
    size = 64 << 20
    for pattern in (1, 2):
        raw = parent.recv()
        region = _native.region_from_bytes(raw)
        regions.append(region)
        ptr = _native.import_region(region, 0)
        dst = torch.zeros(size, dtype=torch.uint8, device="cuda:0")
        rects, n = build_rects([(StridedMem(ptr, (size,), (1,), torch.uint8, 0), StridedMem.from_tensor(dst))])
        _native.copy_rects(0, rects, n)
        _native.stream_sync(0, None)
        assert int(dst.min()) == pattern and int(dst.max()) == pattern
        parent.send("done")
    proc.join(60)
    assert proc.exitcode == 0
    after = _native.import_stats()
    assert regions[0].epoch != regions[1].epoch and regions[0].epoch and regions[1].epoch
    assert bytes(regions[0].ipc_handle) != bytes(regions[1].ipc_handle)
    same_address = regions[0].local_ptr - regions[0].offset == regions[1].local_ptr - regions[1].offset
    if same_address:
        assert after["stale_evictions"] == before["stale_evictions"] + 1
        assert after["live"] == before["live"] + 1
    else:  # the driver happened to place the second allocation elsewhere: both stay mapped
        assert after["live"] == before["live"] + 2
    _native.release_region(regions[1])


def test_export_cache_hits_and_evicts_with_the_storage():
    from torchstore_b200.planner import HbmDescriptor, export_cache

    t = torch.zeros(1 << 20, device="cuda:0")
    h0, m0, e0 = export_cache.hits, export_cache.misses, export_cache.evictions
    a = HbmDescriptor.from_tensor(t)
    b = HbmDescriptor.from_tensor(t)
    assert a == b and export_cache.misses == m0 + 1 and export_cache.hits == h0 + 1
    c = HbmDescriptor.from_tensor(t[1024:])  # another (ptr, nbytes): its own entry, same allocation handle
    assert c.region != a.region and export_cache.misses == m0 + 2
    del t
    assert export_cache.evictions == e0 + 2  # both entries die with the storage


def _allgather_worker(rank, world, port, pg_port, outdir):
    os.environ.update({"RANK": str(rank), "LOCAL_RANK": str(rank), "WORLD_SIZE": str(world), "LOCAL_WORLD_SIZE": str(world),
                       "MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "TORCHSTORE_B200_ALLGATHER": "1"})
    os.environ.pop("TORCHELASTIC_USE_AGENT_STORE", None)
    import torch.distributed as dist
    from torch.distributed.device_mesh import init_device_mesh
    from torch.distributed.tensor import DTensor, Shard

    import torchstore_b200 as ts
    from torchstore_b200.state_dict_utils import _get_rdma_cache

    dev = torch.device("cuda", rank)
    torch.cuda.set_device(dev)

    async def main():
        dist.init_process_group("nccl", init_method=f"tcp://127.0.0.1:{pg_port}", rank=rank, world_size=world, device_id=dev)
        await ts.initialize_spmd(ts.LocalRankStrategy())
        mesh = init_device_mesh("cuda", (world,))
        shapes = {"w": (512, 96), "v": (64,), "u": (128, 4, 8)}
        full = {k: torch.arange(math.prod(s), dtype=torch.float32).reshape(s).to(torch.bfloat16) + i for i, (k, s) in enumerate(shapes.items())}
        src = {k: DTensor.from_local(v.chunk(world, dim=0)[rank].contiguous().to(dev), mesh, (Shard(0),), run_check=False)
               for k, v in full.items()}
        dst = {k: torch.zeros(s, dtype=torch.bfloat16, device=dev) for k, s in shapes.items()}
        await ts.put_state_dict(src, "ag", direct_rdma=True)
        dist.barrier()
        await ts.get_state_dict("ag", user_state_dict=dst, direct_rdma=True)
        ok1 = all(torch.equal(dst[k].cpu(), full[k]) for k in full)
        cl = await ts.client()
        took_nccl = _get_rdma_cache(cl).dests["ag"]._plan is None  # no P2P plan was ever built
        for t in src.values():
            t.to_local().mul_(2.0)
        await ts.put_state_dict(None, "ag", direct_rdma=True)
        dist.barrier()
        await ts.get_state_dict("ag", user_state_dict=dst, direct_rdma=True)
        ok2 = all(torch.equal(dst[k].cpu(), full[k] * 2) for k in full)
        # a layout that is NOT all-gather shaped (one rank wants a column shard) must fall back to P2P on every rank
        dst2 = {"w": torch.zeros(512, 96, dtype=torch.bfloat16, device=dev) if rank == 0 else
                DTensor.from_local(torch.zeros(512, 48, dtype=torch.bfloat16, device=dev), mesh, (Shard(1),), run_check=False, shape=torch.Size((512, 96)), stride=(96, 1))}
        await ts.put_state_dict({"w": src["w"]}, "ag2", direct_rdma=True)
        dist.barrier()
        await ts.get_state_dict("ag2", user_state_dict=dst2, direct_rdma=True)
        got = dst2["w"] if rank == 0 else dst2["w"].to_local()
        want = full["w"] * 2 if rank == 0 else (full["w"] * 2)[:, 48 * rank:48 * (rank + 1)]
        ok3 = torch.equal(got.cpu(), want) and _get_rdma_cache(cl).dests["ag2"]._plan is not None
        dist.barrier()
        await ts.shutdown()
        dist.destroy_process_group()
        np.save(os.path.join(outdir, f"{rank}.npy"), np.array([ok1, took_nccl, ok2, ok3]))

    asyncio.run(main())


@needs2
def test_allgather_route_over_nccl_matches_p2p():
    """BASELINE config #3b's optional route: every rank reads every tensor in full from the ranks' own
    Shard(0) shards -> NCCL all_gather_into_tensor (TORCHSTORE_B200_ALLGATHER=1); any other layout on any
    rank makes ALL ranks take the P2P path (the verdict is min-reduced)."""
    world = 2
    port, pg_port = _free_ports(2)
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_allgather_worker, args=(world, port, pg_port, d), nprocs=world, join=True)
        for r in range(world):
            res = np.load(os.path.join(d, f"{r}.npy"))
            assert res.all(), (r, res)

"""Host tier (SURVEY.md section 8 row f4) on a box WITHOUT a GPU: BASELINE config #1 (single-process
ts.put / ts.get of a 1 MiB fp32 tensor via LocalRankStrategy over POSIX shm) and the reference's
CPU/shm behaviours it pins (tests/test_store.py:27-88,406-455,554-599, tests/test_resharding_basic.py,
tests/test_shared_memory.py): in-place get returns the caller's object, overwrite reuses the segment,
non-contiguous puts, resharded in-place gets, a get without destination is a private copy, deleting a
key unlinks its segment.  Everything goes through the C-ABI (tsb_shm_*, tsb_host_copy_rects)."""

import asyncio
import glob
import os
import time

import pytest
import torch
import torch.multiprocessing as mp

import torchstore_b200 as ts
from torchstore_b200.transport.types import TensorSlice


def run(coro):
    return asyncio.run(coro)


def host_strategy(cls=None, **kw):
    cls = cls or ts.LocalRankStrategy
    return cls(ts.TransportType.SharedMemory, **kw)


@pytest.fixture(autouse=True)
def _env(monkeypatch):
    monkeypatch.delenv("RANK", raising=False)
    monkeypatch.setenv("LOCAL_RANK", "0")
    yield


def _segments():
    return set(glob.glob(f"/dev/shm/tsb200_{os.getpid()}_*"))


def test_config1_one_mib_fp32_put_get_local_rank_strategy():
    """BASELINE.json configs[0]: 512 x 512 fp32 (1 048 576 B), one process, LocalRankStrategy, no GPU."""
    async def main():
        await ts.initialize(num_storage_volumes=1, strategy=host_strategy())
        try:
            t = torch.arange(512 * 512, dtype=torch.float32).reshape(512, 512)
            t0 = time.perf_counter()
            await ts.put("w", t)
            t1 = time.perf_counter()
            got = await ts.get("w")
            t2 = time.perf_counter()
            assert torch.equal(got, t) and got.data_ptr() != t.data_ptr()
            dest = torch.zeros(512, 512)
            out = await ts.get("w", dest)
            assert out is dest and torch.equal(dest, t)
            print(f"config1: put {1e3 * (t1 - t0):.2f} ms, get {1e3 * (t2 - t1):.2f} ms")
            # a get without destination is a private copy: mutating it does not touch the store
            got.zero_()
            assert torch.equal(await ts.get("w"), t)
        finally:
            await ts.shutdown()

    run(main())
    assert not _segments()


def test_overwrite_reuses_segment_and_delete_unlinks_it():
    async def main():
        await ts.initialize(num_storage_volumes=1, strategy=host_strategy())
        try:
            a = torch.randn(300, 70)
            await ts.put("k", a)
            seg1 = _segments()
            assert len(seg1) == 1
            b = torch.randn(300, 70)
            await ts.put("k", b)                      # same shape/dtype: in place, no new segment
            assert _segments() == seg1 and torch.equal(await ts.get("k"), b)
            await ts.put("k", torch.randn(10, 10))     # other shape: new segment, old one released
            seg2 = _segments()
            assert len(seg2) == 1 and seg2 != seg1
            await ts.put("obj", {"x": 1})
            assert await ts.get("obj") == {"x": 1}
            await ts.delete("k")
            import gc

            gc.collect()
            assert not _segments() and not await ts.exists("k")
        finally:
            await ts.shutdown()

    run(main())


def test_non_contiguous_put_and_strided_inplace_get_and_dtypes():
    async def main():
        await ts.initialize(num_storage_volumes=1, strategy=host_strategy())
        try:
            base = torch.arange(64 * 48, dtype=torch.int64).reshape(64, 48)
            view = base.t()[5:40, 3:60:1]                       # non-contiguous source
            await ts.put("nc", view)
            assert torch.equal(await ts.get("nc"), view)
            big = torch.zeros(80, 100, dtype=torch.int64)
            dest = big[10:45, 20:77]                            # strided destination, filled in place
            out = await ts.get("nc", dest)
            assert out is dest and torch.equal(dest, view) and int(big.sum()) == int(view.sum())
            for dt in (torch.bfloat16, torch.float16, torch.uint8, torch.bool, torch.float64):
                x = (torch.rand(33, 17) * 100).to(dt)
                await ts.put(f"d/{dt}", x)
                assert torch.equal(await ts.get(f"d/{dt}"), x)
            s = torch.tensor(3.5)                                # 0-dim
            await ts.put("scalar", s)
            assert (await ts.get("scalar")).item() == 3.5
            # converting in-place get (destination dtype differs): like the reference's copy_
            await ts.put("f", torch.arange(12, dtype=torch.float32).reshape(3, 4))
            d64 = torch.zeros(3, 4, dtype=torch.float64)
            await ts.get("f", d64)
            assert torch.equal(d64, torch.arange(12, dtype=torch.float64).reshape(3, 4))
        finally:
            await ts.shutdown()

    run(main())


def test_resharding_across_volumes_matches_reference_semantics(monkeypatch):
    """FSDP Shard(0) x 4 put from 4 'ranks' into 4 volumes -> TP Shard(1) x 2 in-place gets and a full
    get (reference tests/test_resharding_basic.py:187-277), all on host shm."""
    async def main():
        await ts.initialize(num_storage_volumes=4, strategy=host_strategy())
        try:
            full = torch.arange(512 * 512, dtype=torch.float32).reshape(512, 512)
            for r in range(4):
                monkeypatch.setenv("LOCAL_RANK", str(r))
                shard = full[128 * r:128 * (r + 1)].contiguous()
                cl = await ts.client()
                from torchstore_b200.transport.types import Request

                # a DTensor put, spelt with its slice (no process group on this box)
                req = Request.from_any("w", shard, TensorSlice((128 * r, 0), (r,), (512, 512), (128, 512), (4,)))
                from torchstore_b200.transport import create_transport_buffer

                ref = cl.strategy.select_storage_volume()
                await create_transport_buffer(ref).put_to_storage_volume([req])
                await cl._controller.notify_put_batch.call([req.meta_only()], ref.volume_id)
                if r < 3:
                    with pytest.raises(KeyError, match="partially committed"):
                        await ts.get("w")
            monkeypatch.setenv("LOCAL_RANK", "0")
            for r in range(2):
                dest = torch.zeros(512, 256)
                out = await ts.get("w", dest, TensorSlice((0, 256 * r), (r,), (512, 512), (512, 256), (2,)))
                assert out is dest and torch.equal(dest, full[:, 256 * r:256 * (r + 1)])
            assert torch.equal(await ts.get("w"), full)          # assembled from the 4 stored shards
            part = await ts.get("w", tensor_slice_spec=TensorSlice((100, 7), (0,), (512, 512), (300, 11), (1,)))
            assert torch.equal(part, full[100:400, 7:18])
        finally:
            await ts.shutdown()

    run(main())
    assert not _segments()


def test_state_dict_roundtrip_on_host():
    async def main():
        await ts.initialize(num_storage_volumes=1, strategy=host_strategy())
        try:
            model = torch.nn.Sequential(torch.nn.Linear(32, 64), torch.nn.ReLU(), torch.nn.Linear(64, 8))
            sd = {"model": model.state_dict(), "step": 5}
            await ts.put_state_dict(sd, "v0")
            fresh = await ts.get_state_dict("v0")
            assert fresh["step"] == 5 and all(torch.equal(fresh["model"][k], v) for k, v in sd["model"].items())
            other = torch.nn.Sequential(torch.nn.Linear(32, 64), torch.nn.ReLU(), torch.nn.Linear(64, 8))
            user = {"model": other.state_dict(), "step": 0}
            got = await ts.get_state_dict("v0", user_state_dict=user)
            assert all(got["model"][k] is user["model"][k] and torch.equal(user["model"][k], v) for k, v in sd["model"].items())
        finally:
            await ts.shutdown()

    run(main())


def test_native_host_mover_matches_torch_copy_threaded():
    """tsb_host_copy_rects on strided N-D windows, 1 and 7 threads, against dst.copy_(src)."""
    from torchstore_b200 import _native
    from torchstore_b200.planner import StridedMem, build_rects

    g = torch.Generator().manual_seed(0)
    cases = []
    for shape, sl in (((64, 200, 33), (slice(3, 60), slice(10, 190), slice(0, 33))),
                      ((5000, 300), (slice(0, 5000), slice(17, 211))),
                      ((1 << 22,), (slice(5, (1 << 22) - 3),)),
                      ((40, 40), (slice(0, 40), slice(7, 8)))):
        src = torch.randint(-1000, 1000, shape, dtype=torch.int32, generator=g)
        cases.append((src[sl], shape, sl))
    for threads in (1, 7):
        pairs, checks = [], []
        for sv, shape, sl in cases:
            dst_base = torch.zeros(shape, dtype=torch.int32)
            want = torch.zeros(shape, dtype=torch.int32)
            want[sl].copy_(sv)
            pairs.append((StridedMem.from_tensor(sv), StridedMem.from_tensor(dst_base[sl])))
            checks.append((dst_base, want))
        rects, n = build_rects(pairs)
        _native.host_copy_rects(rects, n, threads)
        assert all(torch.equal(a, b) for a, b in checks)
    # casts are not the host tier's job
    a, b = torch.zeros(8, dtype=torch.float32), torch.zeros(8, dtype=torch.bfloat16)
    rects, n = build_rects([(StridedMem.from_tensor(a), StridedMem.from_tensor(b))])
    with pytest.raises(_native.TsbError):
        _native.host_copy_rects(rects, n, 1)


def _reader(name, nbytes, q):
    from torchstore_b200 import _native

    ptr = _native.shm_attach(name, nbytes)
    import ctypes

    q.put(bytes((ctypes.c_char * 16).from_address(ptr)))
    _native.shm_detach(ptr, nbytes)


def test_segment_is_visible_to_another_process():
    from torchstore_b200 import _native
    import ctypes

    name = f"/tsb200_test_{os.getpid()}"
    ptr = _native.shm_create(name, 4096)
    try:
        ctypes.memmove(ptr, b"0123456789abcdef", 16)
        ctx = mp.get_context("spawn")
        q = ctx.Queue()
        p = ctx.Process(target=_reader, args=(name, 4096, q))
        p.start()
        assert q.get(timeout=60) == b"0123456789abcdef"
        p.join(30)
        with pytest.raises(_native.TsbError):
            _native.shm_create(name, 4096)  # exclusive create
    finally:
        _native.shm_detach(ptr, 4096)
        _native.shm_unlink(name)
    with pytest.raises(_native.TsbError):
        _native.shm_attach(name, 4096)


def test_put_batch_wait_false_on_the_host_tier_completes_inline():
    """wait=False only returns early on the HBM fast lane; other tiers finish the put and hand back a
    PendingPut that is already done (awaiting it is a no-op)."""
    async def main():
        await ts.initialize(num_storage_volumes=1, strategy=host_strategy())
        try:
            pending = await ts.put_batch({"a": torch.ones(4, 4), "o": {"k": 1}}, wait=False)
            assert pending.done
            await pending
            assert torch.equal(await ts.get("a"), torch.ones(4, 4)) and await ts.get("o") == {"k": 1}
        finally:
            await ts.shutdown()

    run(main())


# ---- the reference's own results as the oracle for the host tiers ---------------------------------------
import itertools
import json

import numpy as np

from oracle import reshard_oracle as ro
from tests.helpers import sha256_of
from torchstore_b200.transport import create_transport_buffer
from torchstore_b200.transport.types import Request

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


@pytest.mark.parametrize("transport", ["SharedMemory", "MonarchRPC"])
def test_reshard_matrix_matches_the_reference_results_on_the_host_tiers(transport, monkeypatch):
    """tests/golden/store_reshard.json holds sha256 of what the UNMODIFIED reference (LocalClient +
    SharedMemory transport, run by oracle/gen_golden.py) returned for a matrix of source/destination
    meshes and placements; the host tier and the by-value transport must return the same bytes."""
    gold = json.load(open(os.path.join(GOLDEN, "store_reshard.json")))
    ttype = getattr(ts.TransportType, transport)

    async def put_shard(rank, key, local, tslice):
        monkeypatch.setenv("LOCAL_RANK", str(rank))
        c = await ts.client()
        req = Request(key=key, tensor_val=local, tensor_slice=tslice)
        ref = c.strategy.select_storage_volume()
        await create_transport_buffer(ref).put_to_storage_volume([req])
        await c._controller.notify_put_batch.call([req.meta_only()], ref.volume_id)

    async def main():
        for case in gold["cases"]:
            shape = tuple(case["global_shape"])
            full = torch.arange(int(np.prod(shape)), dtype=torch.float32).reshape(shape)
            smesh, dmesh = tuple(case["src_mesh"]), tuple(case["dst_mesh"])
            spl = [tuple(p) for p in case["src_placements"]]
            dpl = [tuple(p) for p in case["dst_placements"]]
            nvol = max(int(np.prod(smesh)), int(np.prod(dmesh)))
            await ts.initialize(num_storage_volumes=nvol, strategy=ts.LocalRankStrategy(ttype))
            try:
                all_rep = all(p[0] == "R" for p in spl)
                for rank, coord in enumerate(itertools.product(*(range(m) for m in smesh))):
                    sl = ro.make_slice(shape, smesh, coord, spl)
                    local = full[tuple(slice(o, o + s) for o, s in zip(sl.offsets, sl.local_shape))].contiguous()
                    if all_rep:
                        monkeypatch.setenv("LOCAL_RANK", str(rank))
                        await ts.put("test_key", local)
                    else:
                        await put_shard(rank, "test_key", local,
                                        TensorSlice(sl.offsets, sl.coordinates, sl.global_shape, sl.local_shape, sl.mesh_shape))
                for r in case["per_rank"]:
                    coord = list(itertools.product(*(range(m) for m in dmesh)))[r["rank"]]
                    dsl = ro.make_slice(shape, dmesh, coord, dpl)
                    dest = torch.zeros(dsl.local_shape, dtype=torch.float32)
                    monkeypatch.setenv("LOCAL_RANK", str(r["rank"]))
                    got = await ts.get("test_key", dest, TensorSlice(dsl.offsets, dsl.coordinates, dsl.global_shape,
                                                                     dsl.local_shape, dsl.mesh_shape))
                    assert got is dest
                    assert sha256_of(dest) == r["sha256"], (transport, case["src_mesh"], case["dst_mesh"], r["rank"])
                assert sha256_of(await ts.get("test_key")) == case["full_get_sha256"]
            finally:
                await ts.shutdown()

    run(main())
    assert not _segments()


def _leaker(conn):
    from torchstore_b200 import _native

    name = f"/tsb200_{os.getpid()}_1_leak"
    _native.shm_create(name, 4096)
    conn.send(name)  # synchronous: the name is out before we die
    conn.close()
    os._exit(0)      # dies without unlinking, like a killed job


def test_segments_of_dead_processes_are_reaped():
    from torchstore_b200.epoch_board import reap_stale_segments

    ctx = mp.get_context("spawn")
    parent, child = ctx.Pipe()
    p = ctx.Process(target=_leaker, args=(child,))
    p.start()
    assert parent.poll(60)
    name = parent.recv()
    p.join(30)
    assert os.path.exists("/dev/shm" + name)
    mine = f"/tsb200_{os.getpid()}_9_live"
    from torchstore_b200 import _native

    ptr = _native.shm_create(mine, 4096)
    try:
        assert reap_stale_segments() >= 1
        assert not os.path.exists("/dev/shm" + name) and os.path.exists("/dev/shm" + mine)  # live creators are left alone
    finally:
        _native.shm_detach(ptr, 4096)
        _native.shm_unlink(mine)


# ---- the landing-buffer put protocol (transport/buffers.py) on the host tier ----------------------------
async def _handshake_only(ref, key, value):
    """The first phase of a put: the volume hands out (and parks) a landing segment, the client fills it."""
    buf = create_transport_buffer(ref)
    reqs = [Request.from_tensor(key, value)]
    meta = [r.meta_only() for r in reqs]
    assert buf.requires_handshake(reqs)
    await buf.perform_handshake(reqs, meta)
    return buf, meta


def test_concurrent_puts_of_one_key_each_store_their_own_landing_segment():
    """Two puts of the same key both handshake before either one puts: the volume parks each landing
    segment under the put's own nonce, so each put stores the segment its own handshake handed out."""
    import gc

    from torchstore_b200.transport.host import HostVolumeCache

    async def main():
        await ts.initialize(num_storage_volumes=1, strategy=host_strategy())
        try:
            cl = await ts.client()
            ref = cl.strategy.select_storage_volume()
            store = ts.api.rpc._lookup("torchstore/volume/0")[0].store
            values = [torch.full((64, 32), 1.0), torch.full((64, 32), 2.0)]
            puts = []
            for v in values:
                before = _segments()
                buf, meta = await _handshake_only(ref, "k", v)
                puts.append((buf, meta, v, _segments() - before))
            assert all(len(seg) == 1 for *_, seg in puts) and puts[0][3] != puts[1][3]
            for buf, meta, v, seg in puts:
                await ref.volume.put.call(buf, meta)
                stored = store.kv["k"]
                assert torch.equal(stored, v)
                assert {"/dev/shm" + store.transport_context.get(HostVolumeCache).describe(stored).name} == seg
            gc.collect()
            assert _segments() == puts[1][3]  # the first put's segment went with its overwritten value
        finally:
            await ts.shutdown()

    run(main())
    assert not _segments()


def test_abandoned_put_releases_its_landing_segment_after_the_ttl(monkeypatch):
    """A put that handshakes and never puts (its client failed in between) leaves a parked landing
    segment; the first handshake after the TTL releases it, one before the TTL does not, and a reset
    drops whatever is still parked."""
    import gc

    from torchstore_b200.transport import buffers

    async def main():
        await ts.initialize(num_storage_volumes=1, strategy=host_strategy())
        try:
            cl = await ts.client()
            ref = cl.strategy.select_storage_volume()
            await _handshake_only(ref, "lost", torch.ones(128, 64))
            abandoned = _segments()
            assert len(abandoned) == 1
            await ts.put("k", torch.zeros(8))               # a handshake within the TTL keeps it
            gc.collect()
            assert abandoned <= _segments()
            now = buffers.monotonic()
            monkeypatch.setattr(buffers, "monotonic", lambda: now + buffers.LANDING_TTL_S + 1)
            await ts.put("k", torch.ones(8))                # the next handshake after the TTL releases it
            gc.collect()
            assert not abandoned & _segments()
            assert torch.equal(await ts.get("k"), torch.ones(8))
            await _handshake_only(ref, "lost", torch.ones(128, 64))  # parked until the reset below
        finally:
            await ts.shutdown()

    run(main())
    assert not _segments()


@pytest.mark.parametrize("seed", range(3))
def test_store_matches_oracle_across_random_layouts_on_the_host_tier(seed):
    """The differential store harness (tests/store_harness.py) over three host-tier volumes: random
    layouts with uneven, empty and replicated shards, every dtype, and fresh, contiguous, strided and
    converting CPU destinations, each compared with the oracle store; every coverage bucket is reached."""
    from tests.store_harness import run_differential

    async def main():
        await ts.initialize(num_storage_volumes=3, strategy=host_strategy())
        try:
            h = await run_differential(1000 + seed, 40, devices=("cpu",), source_device="cpu")
        finally:
            await ts.shutdown()
        h.assert_coverage()

    run(main())

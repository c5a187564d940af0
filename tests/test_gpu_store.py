"""GPU parity of the store path (ts.put / ts.get / put_state_dict / get_state_dict) against the
fixtures recorded from the reference's LocalClient + SharedMemory transport, plus the behaviours the
reference's integration tests pin (tests/test_store.py, test_tensor_slice.py, test_state_dict.py)."""

import itertools
import json
import os

import numpy as np
import pytest
import torch

import torchstore_b200 as ts
from torchstore_b200 import _native
from oracle import reshard_oracle as ro
from tests.helpers import DEV, run, sha256_of
from torchstore_b200.transport import create_transport_buffer
from torchstore_b200.transport.types import Request, TensorSlice

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(autouse=True)
def _env(monkeypatch):
    monkeypatch.delenv("RANK", raising=False)
    monkeypatch.setenv("LOCAL_RANK", "0")
    monkeypatch.delenv("TORCHSTORE_B200_GET_DEVICE", raising=False)
    yield


async def put_shard(rank, key, local, tslice, monkeypatch):
    """What ts.put(key, dtensor) does on mesh member `rank` (no process group needed)."""
    monkeypatch.setenv("LOCAL_RANK", str(rank))
    c = await ts.client()
    req = Request(key=key, tensor_val=local, tensor_slice=tslice)
    ref = c.strategy.select_storage_volume()
    await create_transport_buffer(ref).put_to_storage_volume([req])
    await c._controller.notify_put_batch.call([req.meta_only()], ref.volume_id)


def test_basic_tensor_put_get_overwrite_and_inplace():
    async def main():
        await ts.initialize()
        try:
            t = torch.randn(512, 512, device=DEV)
            await ts.put("t", t)
            got = await ts.get("t")
            assert got.device.type == "cpu" and torch.equal(got, t.cpu())  # reference: CPU result without a dest
            dest = torch.zeros_like(t)
            out = await ts.get("t", dest)
            assert out is dest and torch.equal(dest, t)
            # overwrite with same shape/dtype reuses the stored buffer
            c = await ts.client()
            vol = ts.api.rpc._lookup("torchstore/volume/0")[0]
            ptr_before = vol.store.kv["t"].data_ptr()
            t2 = t * 3
            await ts.put("t", t2)
            assert vol.store.kv["t"].data_ptr() == ptr_before
            assert torch.equal(await ts.get("t", torch.zeros_like(t)), t2)
            # different shape -> new buffer
            await ts.put("t", torch.ones(4, 4, device=DEV))
            assert torch.equal(await ts.get("t"), torch.ones(4, 4))
            # CPU source and CPU in-place destination ride the copy engine
            h = torch.arange(1000, dtype=torch.int64)
            await ts.put("h", h)
            hd = torch.zeros(1000, dtype=torch.int64)
            assert (await ts.get("h", hd)) is hd and torch.equal(hd, h)
            # non-contiguous put (reference tests/test_store.py:554-599)
            base = torch.randn(64, 48, device=DEV)
            await ts.put("nc", base.t())
            assert torch.equal(await ts.get("nc"), base.t().cpu())
            # get_batch with a mix of in-place / fresh / object
            await ts.put("obj", {"a": 1})
            d2 = torch.zeros(4, 4, device=DEV)
            res = await ts.get_batch({"t": d2, "h": None, "obj": None})
            assert res["t"] is d2 and torch.equal(d2, torch.ones(4, 4, device=DEV))
            assert torch.equal(res["h"], h) and res["obj"] == {"a": 1}
            # result on the GPU when asked
            os.environ["TORCHSTORE_B200_GET_DEVICE"] = "cuda"
            g = await ts.get("h")
            assert g.is_cuda and torch.equal(g.cpu(), h)
            os.environ.pop("TORCHSTORE_B200_GET_DEVICE")
            with pytest.raises(KeyError):
                await ts.get("missing")
            await ts.delete("t")
            assert not await ts.exists("t")
        finally:
            await ts.shutdown()

    run(main())


def test_tensor_slice_gets():
    ts_gold = json.load(open(os.path.join(GOLDEN, "store_reshard.json")))["tensor_slice_get"]

    async def main():
        await ts.initialize()
        try:
            t = torch.arange(100 * 100, dtype=torch.float32, device=DEV).reshape(100, 100)
            await ts.put("t", t)
            spec = TensorSlice(tuple(ts_gold["offsets"]), (), tuple(ts_gold["global_shape"]), tuple(ts_gold["local_shape"]), ())
            got = await ts.get("t", tensor_slice_spec=spec)
            assert sha256_of(got) == ts_gold["sha256"]
            buf = torch.zeros(5, 10, device=DEV)
            out = await ts.get("t", buf, spec)
            assert out is buf and sha256_of(buf) == ts_gold["sha256"]
            with pytest.raises(ValueError, match="does not match"):
                await ts.get("t", torch.zeros(3, 3, device=DEV), spec)
        finally:
            await ts.shutdown()

    run(main())


def test_reshard_matrix_matches_reference(monkeypatch):
    gold = json.load(open(os.path.join(GOLDEN, "store_reshard.json")))

    async def main():
        for case in gold["cases"]:
            shape = tuple(case["global_shape"])
            full = torch.arange(int(np.prod(shape)), dtype=torch.float32).reshape(shape)
            smesh, dmesh = tuple(case["src_mesh"]), tuple(case["dst_mesh"])
            spl = [tuple(p) for p in case["src_placements"]]
            dpl = [tuple(p) for p in case["dst_placements"]]
            nvol = max(int(np.prod(smesh)), int(np.prod(dmesh)))
            await ts.initialize(num_storage_volumes=nvol, strategy=ts.LocalRankStrategy())
            try:
                all_rep = all(p[0] == "R" for p in spl)
                for rank, coord in enumerate(itertools.product(*(range(m) for m in smesh))):
                    sl = ro.make_slice(shape, smesh, coord, spl)
                    local = full[tuple(slice(o, o + s) for o, s in zip(sl.offsets, sl.local_shape))].contiguous().to(DEV)
                    if all_rep:
                        monkeypatch.setenv("LOCAL_RANK", str(rank))
                        await ts.put("test_key", local)
                    else:
                        await put_shard(rank, "test_key", local,
                                        TensorSlice(sl.offsets, sl.coordinates, sl.global_shape, sl.local_shape, sl.mesh_shape),
                                        monkeypatch)
                for r in case["per_rank"]:
                    coord = list(itertools.product(*(range(m) for m in dmesh)))[r["rank"]]
                    dsl = ro.make_slice(shape, dmesh, coord, dpl)
                    dest = torch.zeros(dsl.local_shape, dtype=torch.float32, device=DEV)
                    monkeypatch.setenv("LOCAL_RANK", str(r["rank"]))
                    got = await ts.get("test_key", dest, TensorSlice(dsl.offsets, dsl.coordinates, dsl.global_shape,
                                                                     dsl.local_shape, dsl.mesh_shape))
                    assert got is dest
                    assert sha256_of(dest) == r["sha256"], (case["src_mesh"], case["dst_mesh"], r["rank"])
                whole = await ts.get("test_key")
                assert sha256_of(whole) == case["full_get_sha256"]
            finally:
                await ts.shutdown()

    run(main())


def test_partial_commit_is_not_readable(monkeypatch):
    gold = json.load(open(os.path.join(GOLDEN, "store_reshard.json")))

    async def main():
        await ts.initialize(num_storage_volumes=2, strategy=ts.LocalRankStrategy())
        try:
            small = torch.arange(48, dtype=torch.float32, device=DEV).reshape(8, 6)
            await put_shard(0, "p", small[:4].contiguous(), TensorSlice((0, 0), (0,), (8, 6), (4, 6), (2,)), monkeypatch)
            with pytest.raises(KeyError, match=gold["partial_commit_error_contains"]):
                await ts.get("p")
            assert (await ts.exists("p")) == gold["partial_commit_exists"]
            await put_shard(1, "p", small[4:].contiguous(), TensorSlice((4, 0), (1,), (8, 6), (4, 6), (2,)), monkeypatch)
            assert torch.equal(await ts.get("p"), small.cpu())
        finally:
            await ts.shutdown()

    run(main())


def test_state_dict_roundtrip_inplace_and_fresh():
    async def main():
        await ts.initialize()
        try:
            model = torch.nn.Sequential(torch.nn.Linear(64, 128), torch.nn.ReLU(), torch.nn.Linear(128, 10)).to(DEV)
            sd = {"model": model.state_dict(), "step": 3, "nested": {"lr": 0.1}}
            await ts.put_state_dict(sd, "v0")
            fresh = await ts.get_state_dict("v0")
            assert fresh["step"] == 3 and fresh["nested"] == {"lr": 0.1}
            for k, v in sd["model"].items():
                assert torch.equal(fresh["model"][k], v.cpu())
            other = torch.nn.Sequential(torch.nn.Linear(64, 128), torch.nn.ReLU(), torch.nn.Linear(128, 10)).to(DEV)
            user = {"model": other.state_dict(), "step": 0, "nested": {"lr": 0.0}}
            got = await ts.get_state_dict("v0", user_state_dict=user)
            for k, v in sd["model"].items():
                assert got["model"][k] is user["model"][k] and torch.equal(user["model"][k], v)
        finally:
            await ts.shutdown()

    run(main())


def test_direct_rdma_state_dict_through_api():
    import torch.distributed as dist
    from torch.testing._internal.distributed.fake_pg import FakeStore

    async def main():
        dist.init_process_group("fake", store=FakeStore(), rank=0, world_size=1)
        await ts.initialize()
        try:
            src = {"w": torch.randn(256, 128, device=DEV), "b": torch.randn(128, device=DEV)}
            await ts.put_state_dict(src, "policy", direct_rdma=True)
            assert sorted(await ts.keys()) == ["policy/num_ranks", "policy/rank_0"]
            dst = {"w": torch.zeros(256, 128, device=DEV), "b": torch.zeros(128, device=DEV)}
            out = await ts.get_state_dict("policy", user_state_dict=dst, direct_rdma=True)
            assert out is dst and torch.equal(dst["w"], src["w"]) and torch.equal(dst["b"], src["b"])
            # second round: weights updated in place, no state_dict needed on the source
            src["w"].add_(1.0)
            await ts.put_state_dict(None, "policy", direct_rdma=True)
            await ts.get_state_dict("policy", user_state_dict=dst, direct_rdma=True)
            assert torch.equal(dst["w"], src["w"])
            with pytest.raises(AssertionError, match="user_state_dict is required"):
                await ts.get_state_dict("policy", direct_rdma=True)
            # transfer_dtype: fp32 master -> bf16 destination
            await ts.put_state_dict(src, "policy_bf16", direct_rdma=True, transfer_dtype=torch.bfloat16)
            dst16 = {"w": torch.zeros(256, 128, dtype=torch.bfloat16, device=DEV), "b": torch.zeros(128, dtype=torch.bfloat16, device=DEV)}
            await ts.get_state_dict("policy_bf16", user_state_dict=dst16, direct_rdma=True)
            assert torch.equal(dst16["w"], src["w"].to(torch.bfloat16))
        finally:
            await ts.shutdown()
            dist.destroy_process_group()

    run(main())


def test_volume_memory_is_hbm_arena_and_freed_on_delete():
    async def main():
        await ts.initialize()
        try:
            vol = ts.api.rpc._lookup("torchstore/volume/0")[0]
            await ts.put_batch({f"k{i}": torch.randn(1 << 18, device=DEV) for i in range(8)})
            st = vol.store.stats()
            assert st["slabs"] == 1 and st["in_use"] >= 8 << 20
            assert vol.store.kv["k0"].is_cuda
            await ts.delete_batch([f"k{i}" for i in range(8)])
            import gc

            gc.collect()
            assert vol.store.stats()["in_use"] == 0
        finally:
            await ts.shutdown()

    run(main())


def test_client_fast_lane_replays_put_and_get_and_invalidates_on_layout_change():
    """Store-path fast lane: an identical put_batch / in-place get_batch replays its compiled plan
    (no handshake, no per-key RPC payload); any change of the volume layout (delete, reallocation)
    or of the index drops the session and the slow path takes over -- results stay bit-exact."""
    async def main():
        await ts.initialize()
        try:
            cl = await ts.client()
            lane = cl.fast_lane
            src = {f"w{i}": torch.randn(257, 129, device=DEV) for i in range(6)}
            dst = {k: torch.zeros_like(v) for k, v in src.items()}
            await ts.put_batch(src)                       # slow path, records a session
            assert lane.put_misses == 1 and lane.put_hits == 0 and len(lane.put_sessions) == 1
            before = _native.launch_count()
            for k in src:
                src[k].add_(1.0)
            await ts.put_batch(src)                       # replay
            assert lane.put_hits == 1 and _native.launch_count() == before + 1
            await ts.get_batch(dst)                       # slow get, records
            assert all(torch.equal(dst[k], src[k]) for k in src) and lane.get_hits == 0
            for k in src:
                src[k].mul_(-2.0)
            await ts.put_batch(src)
            out = await ts.get_batch(dst)                 # replayed get: one launch, returns the caller's objects
            assert lane.get_hits == 1 and all(out[k] is dst[k] for k in dst)
            assert all(torch.equal(dst[k], src[k]) for k in src)
            # a different destination set is a different session (not a false hit)
            dst2 = {k: torch.zeros_like(v) for k, v in src.items()}
            await ts.get_batch(dst2)
            assert lane.get_hits == 1 and all(torch.equal(dst2[k], src[k]) for k in src)
            # layout change: delete one key, put it back with another shape -> sessions are stale
            await ts.delete("w0")
            with pytest.raises(Exception):
                await ts.get_batch(dst)                   # w0 is gone: the replay must NOT serve stale bytes
            src["w0"] = torch.randn(300, 10, device=DEV)
            dst["w0"] = torch.zeros(300, 10, device=DEV)
            await ts.put_batch(src)                       # new signature + stale old session
            await ts.get_batch(dst)
            assert all(torch.equal(dst[k], src[k]) for k in src)
            hits = lane.put_hits
            await ts.put_batch(src)                       # and the new batch replays again
            assert lane.put_hits == hits + 1
            # same keys, same shapes, but the volume reallocated (dtype change) -> epoch moved
            src["w1"] = src["w1"].to(torch.float16)
            await ts.put_batch(src)
            got = await ts.get("w1")
            assert got.dtype == torch.float16 and torch.equal(got, src["w1"].cpu())
        finally:
            await ts.shutdown()

    run(main())


def test_failed_recorded_get_batch_caches_no_session_and_destroys_its_plans(monkeypatch):
    """A recorded in-place get_batch that fails after its transports compiled their native plans
    caches no get session and destroys every plan it created."""
    from torchstore_b200.client import LocalClient

    async def main():
        await ts.initialize()
        try:
            cl = await ts.client()
            src = {f"w{i}": torch.randn(65, 33, device=DEV) for i in range(3)}
            await ts.put_batch(src)
            created = []
            real_create = _native.plan_create

            def plan_create(*args, **kwargs):
                created.append(real_create(*args, **kwargs))
                return created[-1]

            async def assemble_fails(self, *args):
                raise RuntimeError("assemble failed")

            monkeypatch.setattr(_native, "plan_create", plan_create)
            monkeypatch.setattr(LocalClient, "_assemble_results", assemble_fails)
            with pytest.raises(RuntimeError, match="assemble failed"):
                await ts.get_batch({k: torch.zeros_like(v) for k, v in src.items()})
            assert created and len(cl.fast_lane.get_sessions) == 0
            for plan in created:
                with pytest.raises(_native.TsbError) as err:
                    _native.plan_info(plan)
                assert err.value.code == _native.TSB_ERR_NOTFOUND
        finally:
            await ts.shutdown()

    run(main())


def test_put_batch_whose_notify_fails_records_no_session(monkeypatch):
    """A put_batch whose notify_put_batch raises leaves its data in the volume but its keys unindexed.
    It must not leave a put session behind: a replay skips the notify, so the identical retry has to
    take the slow path and index the keys."""
    from torchstore_b200 import rpc

    async def main():
        await ts.initialize()
        try:
            cl = await ts.client()
            ctrl = rpc._lookup("torchstore/controller")[0]
            real_notify = ctrl.notify_put_batch
            failed = []

            @rpc.endpoint
            async def notify_fails_once(*args, **kwargs):
                if not failed:
                    failed.append(True)
                    raise RuntimeError("notify lost")
                return await real_notify(*args, **kwargs)

            monkeypatch.setattr(ctrl, "notify_put_batch", notify_fails_once)
            src = {f"n{i}": torch.randn(65, 33, device=DEV) for i in range(3)}
            with pytest.raises(Exception, match="notify lost"):
                await ts.put_batch(src)
            assert cl.fast_lane.put_misses == 1 and len(cl.fast_lane.put_sessions) == 0
            await ts.put_batch(src)                       # slow path again: notifies this time
            assert cl.fast_lane.put_misses == 2 and cl.fast_lane.put_hits == 0
            for k, v in src.items():
                assert torch.equal(await ts.get(k), v.cpu())
        finally:
            await ts.shutdown()

    run(main())


def test_put_batch_wait_false_overlaps_and_completes():
    async def main():
        await ts.initialize()
        try:
            src = {"a": torch.randn(1 << 22, device=DEV), "b": torch.randn(1 << 20, device=DEV)}
            first = await ts.put_batch(src, wait=False)   # first put: completes inline
            assert first.done
            src["a"].add_(3.0)
            pending = await ts.put_batch(src, wait=False)  # replayed: returns with the copy in flight
            marker = torch.ones(1 << 20, device=DEV).sum()  # caller's compute is not fenced behind the copy
            await pending
            assert pending.done and float(marker) == float(1 << 20)
            dst = {k: torch.zeros_like(v) for k, v in src.items()}
            await ts.get_batch(dst)
            assert torch.equal(dst["a"], src["a"]) and torch.equal(dst["b"], src["b"])
        finally:
            await ts.shutdown()

    run(main())


def test_host_destination_of_other_dtype_is_converted_not_overrun():
    """ADVICE r1: stored fp32, caller hands a bf16 / fp64 CPU tensor of the same shape: the raw bytes
    must go through a converting copy (like the reference's copy_), never a memcpy of the stored size."""
    async def main():
        await ts.initialize()
        try:
            x = torch.randn(1000, 37, device=DEV)
            await ts.put("x", x)
            for dt in (torch.bfloat16, torch.float64, torch.float32):
                guard = torch.full((1000 * 37 + 64,), 7.0, dtype=dt)
                dest = guard[:1000 * 37].view(1000, 37)
                out = await ts.get("x", dest)
                assert out is dest and torch.equal(dest, x.cpu().to(dt))
                assert bool((guard[1000 * 37:] == 7.0).all())  # nothing written past the destination
        finally:
            await ts.shutdown()

    run(main())


def test_host_tier_stages_gpu_tensors_like_the_reference():
    """TransportType.SharedMemory chosen explicitly on a GPU box: CUDA tensors go D2H into the (pinned)
    POSIX shm segment and come back H2D, as in the reference (transport/shared_memory.py:374,475); CPU
    destinations are filled by the native host mover.  Never selected by default when CUDA is present."""
    from torchstore_b200.transport import TransportType, get_available_transport

    assert get_available_transport(None) == TransportType.NVLink

    async def main():
        await ts.initialize(num_storage_volumes=1, strategy=ts.LocalRankStrategy(TransportType.SharedMemory))
        try:
            t = torch.randn(777, 129, device=DEV)
            nc = torch.randn(64, 300, device=DEV)[:, 10:200]          # non-contiguous CUDA source
            await ts.put_batch({"t": t, "nc": nc, "o": {"x": 1}})
            vol = ts.api.rpc._lookup("torchstore/volume/0")[0]
            assert not vol.store.kv["t"].is_cuda                        # lives in host shm, not HBM
            got = await ts.get("t")
            assert got.device.type == "cpu" and torch.equal(got, t.cpu())
            dest = torch.zeros(777, 129, device=DEV)
            out = await ts.get("t", dest)
            assert out is dest and torch.equal(dest, t)
            host = torch.zeros(64, 190)
            await ts.get("nc", host)
            assert torch.equal(host, nc.cpu())
            strided = torch.zeros(800, 200, device=DEV)[5:782, 3:132]   # strided CUDA destination
            await ts.get("t", strided)
            assert torch.equal(strided, t)
            t2 = torch.randn(777, 129, device=DEV)
            await ts.put("t", t2)                                       # in-place overwrite of the segment
            assert torch.equal(await ts.get("t"), t2.cpu()) and await ts.get("o") == {"x": 1}
        finally:
            await ts.shutdown()

    run(main())


def test_host_tier_get_into_cuda_lands_after_the_callers_queued_writes():
    """A host-tier get into a contiguous CUDA destination is an H2D copy on the copy stream.  It is
    fenced in behind the caller's stream, so a write the caller queued on the destination before the
    get (a fill behind a sleep) lands first and the fetched data is what remains."""
    from torchstore_b200.transport import TransportType

    async def main():
        await ts.initialize(num_storage_volumes=1, strategy=ts.LocalRankStrategy(TransportType.SharedMemory))
        try:
            t = torch.randn(1024, 1024)
            await ts.put("t", t)
            dest = torch.zeros(1024, 1024, device=DEV)
            torch.cuda.synchronize()
            torch.cuda._sleep(60_000_000)  # clock cycles: ~30 ms on an H100
            dest.fill_(-1)
            out = await ts.get("t", dest)
            torch.cuda.synchronize()
            assert out is dest and torch.equal(dest.cpu(), t)
        finally:
            await ts.shutdown()

    run(main())

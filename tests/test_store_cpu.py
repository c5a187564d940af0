"""Control-plane behaviour on a GPU-less box: objects travel by value through the same
client -> transport -> volume -> controller path as tensors (reference tests/test_store.py,
tests/test_keys.py); the HBM tier refuses to work without a GPU (tensor data on a GPU-less box goes
through the host tier, tests/test_host_tier.py)."""

import asyncio
import os

import pytest
import torch

import torchstore_b200 as ts
from torchstore_b200.controller import Controller, ObjectType, StorageInfo
from torchstore_b200.transport.types import Request, TensorSlice


def run(coro):
    return asyncio.run(coro)


@pytest.fixture(autouse=True)
def _env(monkeypatch):
    monkeypatch.delenv("RANK", raising=False)
    monkeypatch.setenv("LOCAL_RANK", "0")
    yield


def test_objects_roundtrip_keys_exists_delete():
    async def main():
        await ts.initialize()
        try:
            await ts.put("cfg", {"lr": 1e-3, "layers": [1, 2, 3]})
            await ts.put("v0.x", "a")
            await ts.put("v0.y", "b")
            await ts.put("v0.x.z", "c")
            await ts.put("", 0)
            await ts.put(".x", 1)
            assert await ts.get("cfg") == {"lr": 1e-3, "layers": [1, 2, 3]}
            assert sorted(await ts.keys()) == sorted(["cfg", "v0.x", "v0.y", "v0.x.z", "", ".x"])
            assert sorted(await ts.keys("v0")) == ["v0.x", "v0.x.z", "v0.y"]
            assert sorted(await ts.keys("v0.x")) == ["v0.x", "v0.x.z"]
            assert sorted(await ts.keys("")) == ["", ".x"]
            assert await ts.exists("cfg") and not await ts.exists("nope")
            with pytest.raises(KeyError):
                await ts.get("nope")
            assert (await ts.get_batch(["v0.x", "v0.y"])) == {"v0.x": "a", "v0.y": "b"}
            with pytest.raises(ValueError):
                await ts.get_batch([])
            with pytest.raises(ValueError):
                await ts.get_batch(["a", "a"])
            with pytest.raises(AssertionError):
                await ts.put_batch({})
            await ts.delete("cfg")
            assert not await ts.exists("cfg")
            with pytest.raises(Exception):
                await ts.delete("cfg")
            await ts.delete_batch(["v0.x", "missing", "v0.x"])  # idempotent, ignores missing
            assert not await ts.exists("v0.x") and await ts.exists("v0.y")
            await ts.delete_batch([])
            with pytest.raises(TypeError):
                await ts.delete_batch("v0.y")
            # overwrite keeps the kind
            await ts.put("v0.y", {"new": True})
            assert await ts.get("v0.y") == {"new": True}
        finally:
            await ts.shutdown()

    run(main())


def test_multi_volume_local_rank_strategy(monkeypatch):
    async def main():
        await ts.initialize(num_storage_volumes=4, strategy=ts.LocalRankStrategy())
        try:
            for r in range(4):
                monkeypatch.setenv("LOCAL_RANK", str(r))
                await ts.put(f"key_{r:05d}.t1", r + 1)
                await ts.put(f"key_{r:05d}.t2", r + 2)
            assert len(await ts.keys()) == 8
            for r in range(4):
                assert sorted(await ts.keys(f"key_{r:05d}")) == [f"key_{r:05d}.t1", f"key_{r:05d}.t2"]
            monkeypatch.setenv("LOCAL_RANK", "0")
            assert await ts.get("key_00003.t2") == 5  # read from another rank's volume
            monkeypatch.setenv("RANK", "2")  # RANK wins over LOCAL_RANK (reference strategy.py:183-188)
            await ts.put("who", "rank2")
            c = await ts.client()
            vm = await c._controller.locate_volumes.call_one(["who"])
            assert list(vm["who"].keys()) == ["2"]
        finally:
            await ts.shutdown()

    run(main())


def test_initialize_requires_strategy_for_many_volumes():
    with pytest.raises(RuntimeError, match="Must specify controller strategy"):
        run(ts.initialize(num_storage_volumes=2))


def test_state_dict_of_objects_and_missing_mapping():
    async def main():
        await ts.initialize()
        try:
            sd = {"step": 7, "opt": {"lr": 0.1, "betas": (0.9, 0.99)}}
            await ts.put_state_dict(sd, "ckpt")
            assert "ckpt/MAPPING" in await ts.keys()
            got = await ts.get_state_dict("ckpt")
            assert got == sd
            with pytest.raises(RuntimeError, match="Mapping is missing"):
                await ts.get_state_dict("other")
            with pytest.raises(AssertionError):
                await ts.get_state_dict("ckpt", user_state_dict={"different": 1})
            assert await ts.get_state_dict("ckpt", user_state_dict={"different": 1}, strict=False) == sd
        finally:
            await ts.shutdown()

    run(main())


@pytest.mark.skipif(torch.cuda.is_available(), reason="needs a GPU-less box")
def test_hbm_tier_without_gpu_fails_loudly():
    """Asking for the NVLink/HBM transport on a box without a GPU must fail, not degrade."""
    async def main():
        await ts.initialize(num_storage_volumes=1, strategy=ts.ControllerStorageVolumes(ts.TransportType.NVLink))
        try:
            with pytest.raises(Exception, match="no GPU|no CUDA|CUDA"):
                await ts.put("t", torch.zeros(4))
        finally:
            await ts.shutdown()

    run(main())


@pytest.mark.parametrize("kind", ["Gloo", "MonarchRDMA", "TorchComms"])
def test_other_transports_are_rejected(kind):
    async def main():
        await ts.initialize(num_storage_volumes=1, strategy=ts.ControllerStorageVolumes(getattr(ts.TransportType, kind)))
        try:
            with pytest.raises(RuntimeError, match="not part of the torchstore_b200 build"):
                await ts.put("x", 1)
        finally:
            await ts.shutdown()

    run(main())


def test_controller_commit_tracking_and_kind_change():
    """DTensor keys are readable only after every mesh coordinate was put (reference
    controller.py:66-104; tests/test_tensor_slice.py:331-396)."""

    async def main():
        c = Controller()
        c.is_initialized = True

        def req(coord):
            ts_ = TensorSlice((4 * coord, 0), (coord,), (8, 6), (4, 6), (2,))
            return Request(key="w", tensor_slice=ts_)

        await c.notify_put_batch([req(0)], "0")
        with pytest.raises(KeyError, match="partially committed"):
            await c.locate_volumes(["w"])
        assert "w" in await c.locate_volumes(["w"], require_fully_committed=False)
        await c.notify_put_batch([req(1)], "1")
        vm = (await c.locate_volumes(["w"]))["w"]
        assert set(vm) == {"0", "1"} and vm["0"].object_type == ObjectType.TENSOR_SLICE
        with pytest.raises(AssertionError, match="storage type"):
            await c.notify_put_batch([Request(key="w", is_object=True, objects=None)], "0")
        await c.notify_delete("w", "0")
        await c.notify_delete_batch({"1": ["w", "ghost"]})
        with pytest.raises(KeyError, match="Unable to locate"):
            await c.locate_volumes(["w"])
        assert await c.locate_volumes(["w"], missing_ok=True) == {}
        info = StorageInfo(ObjectType.TENSOR)
        with pytest.raises(AssertionError):
            info.update(StorageInfo(ObjectType.OBJECT))

    run(main())


def test_request_from_any_rules():
    t = torch.zeros(3, 4)
    with pytest.raises(ValueError, match="does not match"):
        Request.from_any("k", t, TensorSlice((0, 0), (0,), (8, 8), (2, 2), (1,)))
    with pytest.raises(TypeError):
        Request.from_any("k", "not a tensor")
    r = Request.from_any("k", None, TensorSlice((0, 0), (0,), (8, 8), (2, 2), (1,)))
    assert r.tensor_val is None and r.tensor_slice is not None
    m = Request.from_any("k", t).meta_only()
    assert m.tensor_val is None and m.key == "k"
    a = TensorSlice((0, 0), [0], (8, 8), (2, 2), (1,))
    assert isinstance(a.coordinates, tuple) and hash(a) == hash(TensorSlice((0, 0), (0,), (8, 8), (2, 2), (1,)))


def test_host_strategy_single_volume(monkeypatch):
    monkeypatch.setenv("HOSTNAME", "box-a")

    async def main():
        await ts.initialize(num_storage_volumes=1, strategy=ts.HostStrategy())
        try:
            await ts.put("k", [1, 2, 3])
            assert await ts.get("k") == [1, 2, 3]
            c = await ts.client()
            vm = await c._controller.locate_volumes.call_one(["k"])
            assert list(vm["k"].keys()) == ["box-a"]
            monkeypatch.setenv("HOSTNAME", "box-b")  # a client on another host has no volume here
            with pytest.raises(KeyError, match="No corresponding storage volume"):
                await ts.put("k2", 1)
        finally:
            await ts.shutdown()

    run(main())


def test_rpc_errors_and_mesh():
    from torchstore_b200 import rpc

    class Thing(rpc.Actor):
        def __init__(self, n):
            self.n = n

        @rpc.endpoint
        async def add(self, x):
            return self.n + x

        @rpc.endpoint
        async def boom(self):
            raise KeyError("nope")

        async def hidden(self):
            return 1

    async def main():
        a = rpc.register_actor("t/a", Thing(1))
        b = rpc.register_actor("t/b", Thing(10))
        try:
            assert await a.add.call_one(2) == 3
            with pytest.raises(rpc.ActorError, match="KeyError"):
                await a.boom.call_one()
            with pytest.raises(rpc.ActorError, match="not an endpoint"):
                await a.hidden.call_one()
            mesh = rpc.ActorMesh([({"gpus": 0}, a), ({"gpus": 1}, b)])
            assert await mesh.add.call(5) == [({"gpus": 0}, 6), ({"gpus": 1}, 15)]
            assert await mesh.slice(gpus=1).add.call_one(1) == 11
            with pytest.raises(KeyError):
                mesh.slice(gpus=7)
            with pytest.raises(rpc.ActorError, match="more than one"):
                await mesh.add.call_one(1)
        finally:
            rpc.unregister_actor("t/a")
            rpc.unregister_actor("t/b")
        with pytest.raises(rpc.ActorError, match="no actor named"):
            await a.add.call_one(1)

    run(main())


def test_by_value_actor_rpc_transport(monkeypatch):
    """TransportType.MonarchRPC: payload rides the actor RPC (reference transport/monarch_rpc.py): tensors,
    in-place and strided destinations, resharded gets across two volumes, objects."""
    async def main():
        await ts.initialize(num_storage_volumes=2, strategy=ts.LocalRankStrategy(ts.TransportType.MonarchRPC))
        try:
            t = torch.arange(96, dtype=torch.float32).reshape(8, 12)
            await ts.put("t", t)
            got = await ts.get("t")
            assert torch.equal(got, t) and got.data_ptr() != t.data_ptr()
            big = torch.zeros(10, 20)
            out = await ts.get("t", big[1:9, 4:16])
            assert torch.equal(big[1:9, 4:16], t) and out.data_ptr() == big[1:9, 4:16].data_ptr()
            await ts.put("t", t + 1)                       # overwrite in place on the volume
            assert torch.equal(await ts.get("t"), t + 1)
            await ts.put_batch({"o": {"a": 1}, "u": torch.ones(3, dtype=torch.int64)})
            assert (await ts.get_batch(["o", "u"]))["o"] == {"a": 1}
            from torchstore_b200.transport import create_transport_buffer

            for r in range(2):
                monkeypatch.setenv("LOCAL_RANK", str(r))
                cl = await ts.client()
                req = Request.from_any("w", t[4 * r:4 * r + 4].contiguous(), TensorSlice((4 * r, 0), (r,), (8, 12), (4, 12), (2,)))
                ref = cl.strategy.select_storage_volume()
                await create_transport_buffer(ref).put_to_storage_volume([req])
                await cl._controller.notify_put_batch.call([req.meta_only()], ref.volume_id)
            assert torch.equal(await ts.get("w"), t)
            col = torch.zeros(8, 6)
            await ts.get("w", col, TensorSlice((0, 6), (1,), (8, 12), (8, 6), (2,)))
            assert torch.equal(col, t[:, 6:])
        finally:
            await ts.shutdown()

    run(main())

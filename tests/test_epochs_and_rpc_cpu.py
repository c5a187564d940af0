"""Host-side logic added in round 2, on the CPU: layout/index epochs that guard the store fast lane,
the per-actor mailbox (one endpoint at a time without blocking an event loop), nonce-keyed pending puts."""

import asyncio
import threading
import time

import pytest
import torch

import torchstore_b200 as ts
from torchstore_b200 import rpc
from torchstore_b200.controller import Controller
from torchstore_b200.transport.types import Request, TensorSlice


def run(coro):
    return asyncio.run(coro)


@pytest.fixture(autouse=True)
def _env(monkeypatch):
    monkeypatch.delenv("RANK", raising=False)
    monkeypatch.setenv("LOCAL_RANK", "0")
    yield


def test_controller_epoch_moves_only_when_the_index_changes_shape():
    async def main():
        c = Controller()
        c.is_initialized = True
        e0 = await c.get_epoch()
        r = Request(key="k")
        await c.notify_put_batch([r], "0")
        e1 = await c.get_epoch()
        assert e1 > e0
        await c.notify_put_batch([r], "0")            # overwrite of an indexed key: unchanged
        assert await c.get_epoch() == e1
        s0 = Request(key="w", tensor_slice=TensorSlice((0, 0), (0,), (8, 4), (4, 4), (2,)))
        s1 = Request(key="w", tensor_slice=TensorSlice((4, 0), (1,), (8, 4), (4, 4), (2,)))
        await c.notify_put_batch([s0], "0")
        e2 = await c.get_epoch()
        await c.notify_put_batch([s0], "0")
        assert await c.get_epoch() == e2
        await c.notify_put_batch([s1], "0")            # a new slice of a known key
        e3 = await c.get_epoch()
        assert e3 > e2
        await c.notify_put_batch([s1], "1")            # a new volume for a known key
        e4 = await c.get_epoch()
        assert e4 > e3
        await c.notify_delete("k", "0")
        assert await c.get_epoch() > e4

    run(main())


def test_volume_layout_epoch_ignores_in_place_overwrites():
    """Through the host tier (no GPU here): same semantics as the HBM volumes."""
    async def main():
        await ts.initialize(num_storage_volumes=1, strategy=ts.LocalRankStrategy(ts.TransportType.SharedMemory))
        try:
            vol = rpc._lookup("torchstore/volume/0")[0]
            e0 = vol.store.epoch
            await ts.put("a", torch.zeros(16, 16))
            e1 = vol.store.epoch
            assert e1 > e0
            await ts.put("a", torch.ones(16, 16))      # same shape/dtype: stored buffer reused
            assert vol.store.epoch == e1
            await ts.put("a", torch.ones(4, 4))        # reallocation
            e2 = vol.store.epoch
            assert e2 > e1
            await ts.put("o", {"x": 1})
            e3 = vol.store.epoch
            await ts.put("o", {"x": 2})                # objects: same kind, same key -> unchanged
            assert vol.store.epoch == e3 > e2
            await ts.delete("a")
            assert vol.store.epoch > e3
            assert await vol.epoch() == vol.store.epoch
        finally:
            await ts.shutdown()

    run(main())


def test_mailbox_serialises_endpoints_across_loops_without_blocking_them():
    class Counter(rpc.Actor):
        def __init__(self):
            self.inside = 0
            self.max_inside = 0
            self.calls = 0

        @rpc.endpoint
        async def work(self, delay):
            self.inside += 1
            self.max_inside = max(self.max_inside, self.inside)
            await asyncio.sleep(delay)          # yields: another coroutine could enter without the mailbox
            self.inside -= 1
            self.calls += 1
            return self.calls

    ref = rpc.register_actor("t/counter", Counter())
    other = rpc.register_actor("t/other", Counter())
    try:
        async def same_loop():
            # two coroutines of ONE loop calling the same actor: strictly one at a time, and the loop
            # keeps serving a different actor meanwhile (an RLock would let both in / a plain lock would hang)
            t0 = time.perf_counter()
            res = await asyncio.gather(ref.work.call_one(0.05), ref.work.call_one(0.05), other.work.call_one(0.01))
            return res, time.perf_counter() - t0

        res, dt = run(same_loop())
        obj = rpc._lookup("t/counter")[0]
        assert obj.max_inside == 1 and sorted(res[:2]) == [1, 2] and dt >= 0.095

        # a second thread with its own loop contends for the same mailbox
        out = []

        def worker():
            out.append(asyncio.run(ref.work.call_one(0.03)))

        th = threading.Thread(target=worker)

        async def main_side():
            th.start()
            return await ref.work.call_one(0.03)

        mine = run(main_side())
        th.join(10)
        assert obj.max_inside == 1 and sorted([mine, out[0]]) == [3, 4]
    finally:
        rpc.unregister_actor("t/counter")
        rpc.unregister_actor("t/other")


def test_remote_calls_overlap_instead_of_freezing_the_loop():
    """asyncio.gather over two remote endpoints really is concurrent (socket I/O runs off-loop)."""
    class Slow(rpc.Actor):
        @rpc.endpoint
        async def nap(self, s):
            await asyncio.sleep(s)
            return s

    server = rpc.ActorServer.instance()
    a = rpc.register_actor("t/slow_a", Slow())
    b = rpc.register_actor("t/slow_b", Slow())
    try:
        ra = rpc.RemoteActorRef(server.address, server.authkey, "t/slow_a")
        rb = rpc.RemoteActorRef(server.address, server.authkey, "t/slow_b")

        async def main():
            ticks = 0

            async def ticker():
                nonlocal ticks
                for _ in range(20):
                    await asyncio.sleep(0.005)
                    ticks += 1

            t0 = time.perf_counter()
            res = await asyncio.gather(ra.nap.call_one(0.1), rb.nap.call_one(0.1), ticker())
            return res, time.perf_counter() - t0, ticks

        res, dt, ticks = run(main())
        assert res[:2] == [0.1, 0.1] and ticks == 20   # the caller's loop stayed live
        assert dt < 0.35                                 # one connection serialises its requests, the loop is not frozen
        assert a is not None and b is not None
    finally:
        rpc.unregister_actor("t/slow_a")
        rpc.unregister_actor("t/slow_b")


def test_double_initialize_is_refused_before_touching_the_live_store():
    async def main():
        await ts.initialize(num_storage_volumes=1, strategy=ts.LocalRankStrategy(ts.TransportType.SharedMemory))
        try:
            await ts.put("keep", torch.arange(10.0))
            with pytest.raises(RuntimeError, match="already initialized"):
                await ts.initialize(num_storage_volumes=1, strategy=ts.LocalRankStrategy(ts.TransportType.SharedMemory))
            assert torch.equal(await ts.get("keep"), torch.arange(10.0))   # data survived the bad call
        finally:
            await ts.shutdown()

    run(main())


def test_epoch_board_mirrors_controller_and_volume_epochs_in_shared_memory():
    import glob
    import os

    from torchstore_b200 import epoch_board

    async def main():
        await ts.initialize(num_storage_volumes=2, strategy=ts.LocalRankStrategy(ts.TransportType.SharedMemory))
        try:
            cl = await ts.client()
            name, slots = cl.strategy.epoch_board
            assert sorted(slots) == ["0", "1"] and sorted(slots.values()) == [1, 2]
            assert os.path.exists("/dev/shm" + name)
            board = epoch_board.attached(name)
            vol0 = rpc._lookup("torchstore/volume/0")[0]
            ctrl = rpc._lookup("torchstore/controller")[0]
            assert board.read(0) == ctrl.epoch and board.read(slots["0"]) == vol0.store.epoch
            await ts.put("a", torch.zeros(8))
            assert board.read(0) == ctrl.epoch > 0 and board.read(slots["0"]) == vol0.store.epoch > 0
            before = (board.read(0), board.read(slots["0"]))
            await ts.put("a", torch.ones(8))                       # in place: neither epoch moves
            assert (board.read(0), board.read(slots["0"])) == before
            await ts.delete("a")
            assert board.read(0) > before[0] and board.read(slots["0"]) > before[1]
            assert board.read(slots["1"]) == rpc._lookup("torchstore/volume/1")[0].store.epoch
            # a StorageVolumeRef carries the board so transports can find their slot
            assert cl.strategy.get_storage_volume("1").epoch_board == (name, slots)
            return name
        finally:
            await ts.shutdown()

    name = run(main())
    assert not os.path.exists("/dev/shm" + name) and not glob.glob("/dev/shm/tsb200_epochs_*")


def test_epoch_board_also_serves_the_default_single_volume_store():
    async def main():
        await ts.initialize(num_storage_volumes=1, strategy=ts.ControllerStorageVolumes(ts.TransportType.SharedMemory))
        try:
            cl = await ts.client()
            assert cl.strategy.epoch_board is not None and list(cl.strategy.epoch_board[1].values()) == [1]
        finally:
            await ts.shutdown()

    run(main())

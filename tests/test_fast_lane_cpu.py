"""The store fast lane on the CPU (fast_lane.py): the session cache, when a session is dropped, what a
recording keeps, and which batches have a signature.  Fakes stand in for native plans and transports."""

import asyncio

import torch

from torchstore_b200.transport.types import Request, TensorSlice


def run(coro):
    return asyncio.run(coro)


def test_session_lru_closes_what_it_replaces_evicts_drops_and_clears():
    """The fast lane's put and get sessions hold native plans: every session leaving the cache is closed."""
    from torchstore_b200.fast_lane import SessionLRU

    class Sess:
        closed = False

        def close(self):
            self.closed = True

    lru = SessionLRU(2)
    a, b, c, a2 = Sess(), Sess(), Sess(), Sess()
    lru.put("a", a)
    lru.put("b", b)
    assert lru.get("a") is a                 # a becomes the most recently used
    lru.put("c", c)                          # over the cap: b, the least recently used, goes
    assert b.closed and not a.closed and not c.closed and len(lru) == 2 and lru.get("b") is None
    lru.put("a", a2)                         # replacing a signature closes the old session
    assert a.closed and lru.get("a") is a2
    lru.drop("c")
    assert c.closed and len(lru) == 1
    lru.clear()
    assert a2.closed and len(lru) == 0


class _FakePlans:
    def __init__(self):
        self.closed = False
        self.launches = []

    def launch(self, fence_out=True):
        self.launches.append(fence_out)

    async def wait(self):
        pass

    def close(self):
        self.closed = True


class _FakePart:
    """Stands in for fast_lane.Part: one volume's plans and whether its layout epoch still holds."""

    def __init__(self, ok=True):
        self.plans = _FakePlans()
        self.ok = ok
        self.closed = False

    async def valid(self):
        return self.ok

    def close(self):
        self.closed = True


class _FakeController:
    def __init__(self, epoch):
        self.epoch = epoch
        outer = self

        class _GetEpoch:
            async def call_one(self):
                return outer.epoch

        self.get_epoch = _GetEpoch()


class _FakeTransport:
    """Stands in for a fast-lane transport: compiled plans, handed over with the epoch they were built
    under, or closed when the request got no epoch."""

    supports_fast_lane = True

    def __init__(self, volume_id, epoch=7, compiles=True):
        from types import SimpleNamespace

        self.storage_volume_ref = SimpleNamespace(volume_id=volume_id)
        self.record = False
        self.epoch = epoch
        self.plans = _FakePlans() if compiles else None

    def take_recorded(self):
        if self.plans is not None and self.epoch is None:
            self.plans.close()
            return None
        return None if self.plans is None else (self.plans, self.epoch)


def test_fast_lane_drops_and_closes_sessions_whose_epochs_moved():
    from types import SimpleNamespace

    from torchstore_b200.fast_lane import FastLane, Session

    async def main():
        ctrl = _FakeController(epoch=5)
        lane = FastLane(ctrl, SimpleNamespace(epoch_board=None))
        put = _FakePart()
        lane.put_sessions.put("p", Session([put]))
        assert await lane.replay_put("p") is put.plans and put.plans.launches == [False]  # no fence-out
        put.ok = False                                   # the volume reallocated a key of the batch
        assert await lane.replay_put("p") is None and put.closed and len(lane.put_sessions) == 0
        assert (lane.put_hits, lane.put_misses) == (1, 1)

        dst = torch.zeros(4)
        parts = [_FakePart(), _FakePart()]
        lane.get_sessions.put("g", Session(parts, controller_epoch=5, final={"k": dst}))
        out = await lane.replay_get("g")
        assert out == {"k": dst} and out["k"] is dst and all(p.plans.launches == [True] for p in parts)
        ctrl.epoch = 6                                   # the index changed shape
        assert await lane.replay_get("g") is None and all(p.closed for p in parts)
        assert len(lane.get_sessions) == 0 and lane.get_hits == 1

        parts = [_FakePart(), _FakePart(ok=False)]       # one volume's layout moved
        lane.get_sessions.put("g", Session(parts, controller_epoch=6, final={"k": dst}))
        assert await lane.replay_get("g") is None and all(p.closed for p in parts)
        assert len(lane.get_sessions) == 0 and lane.get_hits == 1

    run(main())


def test_fast_lane_keeps_only_recordings_that_succeeded_in_place():
    from types import SimpleNamespace

    from torchstore_b200.fast_lane import FastLane

    async def main():
        lane = FastLane(_FakeController(epoch=3), SimpleNamespace(epoch_board=None))
        dst = {"a": torch.zeros(4), "b": torch.zeros(4)}
        requests = [Request.from_any(k, v) for k, v in dst.items()]

        async def recorded_get(*transports):
            rec = await lane.record_get("g")
            rec.attach(list(transports))
            assert all(t.record for t in transports)
            return rec

        # failed get (no result): every plan closed, nothing cached
        ts_ = [_FakeTransport("0"), _FakeTransport("1")]
        lane.finish_get(await recorded_get(*ts_), requests, None, None)
        assert all(t.plans.closed for t in ts_) and len(lane.get_sessions) == 0
        # one result did not land in the caller's tensor (a host copy): nothing cached
        ts_ = [_FakeTransport("0"), _FakeTransport("1")]
        results = {"a": dst["a"], "b": torch.zeros(4)}
        lane.finish_get(await recorded_get(*ts_), requests, results, dict(dst))
        assert all(t.plans.closed for t in ts_) and len(lane.get_sessions) == 0
        # one volume compiled nothing (D2H results): the other's plans are closed
        ts_ = [_FakeTransport("0"), _FakeTransport("1", compiles=False)]
        lane.finish_get(await recorded_get(*ts_), requests, dict(dst), dict(dst))
        assert ts_[0].plans.closed and len(lane.get_sessions) == 0
        # a failed request has no volume epoch
        ts_ = [_FakeTransport("0"), _FakeTransport("1", epoch=None)]
        lane.finish_get(await recorded_get(*ts_), requests, dict(dst), dict(dst))
        assert all(t.plans.closed for t in ts_) and len(lane.get_sessions) == 0
        # in place and successful: kept, with a copy of the caller's result dict
        ts_ = [_FakeTransport("0"), _FakeTransport("1")]
        final = dict(dst)
        lane.finish_get(await recorded_get(*ts_), requests, dict(dst), final)
        sess = lane.get_sessions.get("g")
        assert not any(t.plans.closed for t in ts_) and sess.controller_epoch == 3
        assert sess.final == final and sess.final is not final

        # a put that failed (or whose notify failed) closes its plans and caches nothing
        from torchstore_b200.fast_lane import Recording

        t = _FakeTransport("0")
        rec = Recording(("0",))
        rec.attach([t])
        lane.commit(rec, ok=False)
        assert t.record and t.plans.closed and len(lane.put_sessions) == 0
        t = _FakeTransport("0")
        rec = Recording(("0",))
        rec.attach([t])
        lane.commit(rec, ok=True)
        assert not t.plans.closed and len(lane.put_sessions) == 1

        # a transport without the lane: nothing records
        plain = SimpleNamespace(supports_fast_lane=False, record=False)
        rec = Recording(("0",))
        rec.attach([_FakeTransport("0"), plain])
        assert rec.transports == [] and not plain.record

    run(main())


def test_fast_lane_signature_needs_a_cuda_tensor_per_request(monkeypatch):
    from torchstore_b200.fast_lane import signature

    class CudaLike:
        """Just enough of a CUDA tensor for a signature."""

        is_cuda = True
        shape = (4, 2)
        dtype = torch.float32

        def data_ptr(self):
            return 4096

        def stride(self):
            return (2, 1)

    gpu = Request(key="a", tensor_val=CudaLike())
    sl = TensorSlice((0, 0), (0,), (8, 2), (4, 2), (2,))
    sliced = Request(key="s", tensor_val=CudaLike(), tensor_slice=sl)
    assert signature([gpu]) == (("a", None, 4096, (4, 2), (2, 1), torch.float32),)
    assert signature([gpu, sliced], "vol0") == ("vol0", signature([gpu])[0], ("s", sl, 4096, (4, 2), (2, 1), torch.float32))
    assert signature([gpu, Request.from_objects("o", {"x": 1})]) is None      # an object
    assert signature([gpu, Request.from_any("c", torch.zeros(4, 2))]) is None  # a CPU tensor
    assert signature([gpu, Request.from_any("m", None)]) is None              # no destination
    monkeypatch.setenv("TORCHSTORE_B200_FAST_LANE", "0")
    assert signature([gpu]) is None

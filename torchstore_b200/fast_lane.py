"""The store path's fast lane (DESIGN.md §4): a ``put_batch`` or in-place ``get_batch`` that repeats an
earlier batch (same keys, slices and client memory) replays the native plans that batch compiled, while
the epochs it was recorded under hold: its volumes' layout epochs, and for a get the controller's index
epoch its volume map was read under.  This module is the only code that knows which batches replay and
when a recording becomes a session; a transport only compiles plans while its ``record`` flag is set."""

from __future__ import annotations

import asyncio
import collections
import os
from dataclasses import dataclass, field
from typing import Any

import torch

from torchstore_b200 import epoch_board
from torchstore_b200.launch import Plans


def signature(requests: list, volume_id: str | None = None) -> tuple | None:
    """Identity of a batch: keys, wanted slices and client memory, prefixed with the volume id for a
    put.  None when the lane is off or a request has no CUDA tensor (nothing to replay from or into)."""
    if os.environ.get("TORCHSTORE_B200_FAST_LANE", "1") != "1":
        return None
    sig = [] if volume_id is None else [volume_id]
    for r in requests:
        t = r.tensor_val
        if r.is_object or t is None or not t.is_cuda:
            return None
        sig.append((r.key, r.tensor_slice, t.data_ptr(), tuple(t.shape), tuple(t.stride()), t.dtype))
    return tuple(sig)


class SessionLRU:
    """Replayable sessions keyed by signature, least recently used first.  A session is closed when
    it is replaced, dropped, evicted past ``cap`` or cleared."""

    def __init__(self, cap: int) -> None:
        self.cap = cap
        self._by_sig: "collections.OrderedDict[object, object]" = collections.OrderedDict()

    def __len__(self) -> int:
        return len(self._by_sig)

    def get(self, sig):
        sess = self._by_sig.get(sig)
        if sess is not None:
            self._by_sig.move_to_end(sig)
        return sess

    def put(self, sig, sess) -> None:
        self.drop(sig)
        self._by_sig[sig] = sess
        while len(self._by_sig) > self.cap:
            self._by_sig.popitem(last=False)[1].close()

    def drop(self, sig) -> None:
        sess = self._by_sig.pop(sig, None)
        if sess is not None:
            sess.close()

    def clear(self) -> None:
        for sess in self._by_sig.values():
            sess.close()
        self._by_sig.clear()


@dataclass
class Part:
    """One volume's share of a session: its compiled plans and the volume layout epoch they were built
    under.  While that epoch is unchanged no key of the batch has moved on the volume."""

    plans: Plans
    epoch: int
    volume_ref: Any
    board: Any = None   # (EpochBoard, slot): read the volume's epoch from shared memory instead of by RPC

    async def valid(self) -> bool:
        if self.board is not None:
            return self.board[0].read(self.board[1]) == self.epoch
        return await self.volume_ref.volume.epoch.call_one() == self.epoch

    def close(self) -> None:
        self.plans.close()


@dataclass
class Session:
    parts: list                          # Part per volume (a put has one)
    controller_epoch: int | None = None  # get: the index epoch its volume map was read under
    final: dict | None = None            # get: key -> the caller's destination object

    def close(self) -> None:
        for p in self.parts:
            p.close()


@dataclass
class Recording:
    """A slow-path batch whose transports compile plans, to become a session if it succeeds."""

    sig: tuple
    controller_epoch: int | None = None
    transports: list = field(default_factory=list)

    def attach(self, transports: list) -> None:
        """Record through ``transports`` when every one of them supports the lane."""
        if all(t.supports_fast_lane for t in transports):
            for t in transports:
                t.record = True
            self.transports = transports


class FastLane:
    """One client's put and get sessions and their counters."""

    def __init__(self, controller, strategy) -> None:
        self._controller = controller
        # (shm name, {volume id: slot}), published by the controller before any client exists
        self._board_name, self._board_slots = getattr(strategy, "epoch_board", None) or (None, {})
        cap = int(os.environ.get("TORCHSTORE_B200_MAX_SESSIONS", "64"))
        self.put_sessions = SessionLRU(cap)
        self.get_sessions = SessionLRU(cap)
        self.put_hits = self.put_misses = self.get_hits = 0

    async def replay_put(self, sig: tuple) -> Plans | None:
        """Launch the put recorded under ``sig`` if its volume layout is unchanged, and return its plans
        to await; no fence-out, since the copy only reads the caller's memory.  None is a miss."""
        sess = self.put_sessions.get(sig)
        if sess is not None:
            part = sess.parts[0]
            if await part.valid():
                self.put_hits += 1
                part.plans.launch(fence_out=False)
                return part.plans
            self.put_sessions.drop(sig)
        self.put_misses += 1
        return None

    async def replay_get(self, sig: tuple) -> dict | None:
        """Run the get recorded under ``sig`` if neither the index nor a volume layout has changed;
        returns the caller's destination objects, or None."""
        sess = self.get_sessions.get(sig)
        if sess is None:
            return None
        board = epoch_board.attached(self._board_name)
        if board is not None:
            got = [board.read(0)] + [await p.valid() for p in sess.parts]  # memory loads, no RPC
        else:
            got = await asyncio.gather(self._controller.get_epoch.call_one(), *[p.valid() for p in sess.parts])
        if got[0] != sess.controller_epoch or not all(got[1:]):
            self.get_sessions.drop(sig)
            return None
        for p in sess.parts:
            p.plans.launch()
        for p in sess.parts:
            await p.plans.wait()
        self.get_hits += 1
        return dict(sess.final)

    async def record_get(self, sig: tuple) -> Recording | None:
        """Read the controller epoch BEFORE the volume map: if the index changes in between, the session
        is born stale (and is dropped on its first replay) rather than wrongly valid."""
        try:
            board = epoch_board.attached(self._board_name)
            epoch = board.read(0) if board is not None else await self._controller.get_epoch.call_one()
        except Exception:
            return None
        return Recording(sig, epoch)

    def finish_get(self, rec: Recording, requests: list, results: dict | None, final: dict | None) -> None:
        """A get replays only if it succeeded (``final`` is set) and every result landed in place."""
        ok = final is not None and all(
            isinstance(results[r.key], torch.Tensor) and results[r.key].data_ptr() == r.tensor_val.data_ptr()
            for r in requests)
        self.commit(rec, ok, dict(final) if ok else None)

    def commit(self, rec: Recording, ok: bool, final: dict | None = None) -> None:
        """Keep a recording that succeeded as a session if every transport compiled plans under a volume
        epoch; otherwise close every plan it compiled.  A put (no controller epoch) is ``ok`` only once
        the controller's notify has returned too, since a replay skips the notify."""
        lru = self.put_sessions if rec.controller_epoch is None else self.get_sessions
        parts = [self._part(t) for t in rec.transports]
        if ok and parts and all(p is not None for p in parts):
            lru.put(rec.sig, Session(parts, rec.controller_epoch, final))
            return
        for p in parts:
            if p is not None:
                p.close()

    def _part(self, transport) -> Part | None:
        recorded = transport.take_recorded()
        if recorded is None:
            return None
        ref = transport.storage_volume_ref
        board = epoch_board.attached(self._board_name)
        slot = self._board_slots.get(ref.volume_id)
        return Part(*recorded, ref, (board, slot) if board is not None and slot is not None else None)

    def clear(self) -> None:
        """Close every session and drop this process's epoch-board attachment (store shutdown)."""
        self.put_sessions.clear()
        self.get_sessions.clear()
        epoch_board.forget(self._board_name)

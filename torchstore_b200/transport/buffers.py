"""The transport plugin contract (reference torchstore/transport/buffers.py:20-361).

A ``TransportBuffer`` is created by the client for one (client, volume) pair, runs its client half
in the caller's process, is pickled into the volume RPCs and runs its volume half there.  The
lifecycle below is the reference's, less the hooks no transport of this build uses:

PUT   requires_handshake? -> perform_handshake (volume: recv_handshake; client: _post_handshake)
      -> _pre_put_hook -> RPC volume.put (volume: handle_put_request; returns the layout epoch)
      -> drop (always)
GET   _pre_get_hook -> RPC volume.get (volume: handle_get_request; the buffer object comes back with
      the layout epoch the store stamped on it) -> _handle_storage_volume_response -> drop (always)

``LandingBufferTransport`` below is the two-phase put both data tiers share (``transport/hbm.py``,
``transport/host.py``); ``transport/actor_rpc.py`` carries its payload by value instead.
"""

from __future__ import annotations

import os
from abc import ABC, abstractmethod
from collections.abc import Iterable
from dataclasses import dataclass
from time import monotonic
from typing import TYPE_CHECKING, Any, TypeVar

import torch

from torchstore_b200.logging import LatencyTracker
from torchstore_b200.transport.types import Request

if TYPE_CHECKING:
    from torchstore_b200.strategy import StorageVolumeRef


class TransportCache(ABC):
    """Long-lived per-transport state kept in a TransportContext."""

    def delete(self, keys: set[str]) -> None:  # most caches are not keyed by store key
        return

    @abstractmethod
    def clear(self) -> None: ...


T = TypeVar("T", bound=TransportCache)


class TransportContext:
    """Type-keyed registry of transport caches, created lazily on first ``get``."""

    def __init__(self) -> None:
        self._caches: dict[type[TransportCache], TransportCache] = {}

    def get(self, cache_type: type[T]) -> T:
        cache = self._caches.get(cache_type)
        if cache is None:
            cache = self._caches[cache_type] = cache_type()
        return cache  # type: ignore[return-value]

    def clear(self) -> None:
        for cache in self._caches.values():
            cache.clear()
        self._caches.clear()

    def delete(self, keys: str | Iterable[str]) -> None:
        key_set = {keys} if isinstance(keys, str) else set(keys)
        if key_set:
            for cache in self._caches.values():
                cache.delete(key_set)


class TransportBuffer:
    """Base class; subclasses implement the volume handlers and the response handler."""

    supports_batch_puts: bool = False
    supports_batch_gets: bool = False
    supports_strided_inplace: bool = False  # in-place destinations may be non-contiguous views
    supports_fast_lane: bool = False        # has a ``record`` flag and ``take_recorded`` (fast_lane.py)

    def __init__(self, storage_volume_ref: "StorageVolumeRef"):
        self.storage_volume_ref = storage_volume_ref
        # the volume's layout epoch (storage_volume.py): returned by a put, stamped on a get's buffer
        self._volume_epoch = None

    def __getstate__(self) -> dict[str, Any]:
        state = self.__dict__.copy()
        state["storage_volume_ref"] = None  # process-local handle
        return state

    # ---- client side ----------------------------------------------------------------------------
    def requires_handshake(self, requests: list[Request]) -> bool:
        """Puts only: whether the volume is asked where the data goes before the put RPC."""
        return False

    async def put_to_storage_volume(self, requests: list[Request]) -> None:
        batches = [requests] if self.supports_batch_puts else [[r] for r in requests]
        for batch in batches:
            await self._put_requests(batch)

    async def _put_requests(self, requests: list[Request]) -> None:
        tracker = LatencyTracker("put")
        meta = [r.meta_only() for r in requests]
        try:
            if self.requires_handshake(requests):
                await self.perform_handshake(requests, meta, tracker)
            await self._pre_put_hook(requests)
            tracker.track_step("_pre_put_hook")
            self._volume_epoch = await self.storage_volume_ref.volume.put.call(self, meta)
            tracker.track_step("volume.put.call")
        finally:
            await self.drop()
            tracker.track_step("drop")
            tracker.track_e2e()

    async def get_from_storage_volume(self, requests: list[Request]) -> list[Any]:
        if self.supports_batch_gets:
            return await self._get_requests(requests)
        out: list[Any] = []
        for r in requests:
            out.extend(await self._get_requests([r]))
        return out

    async def _get_requests(self, requests: list[Request]) -> list[Any]:
        tracker = LatencyTracker("get")
        meta = [r.meta_only() for r in requests]
        try:
            await self._pre_get_hook(requests)
            tracker.track_step("_pre_get_hook")
            returned = await self.storage_volume_ref.volume.get.call_one(self, meta)
            response = await self._handle_storage_volume_response(requests, returned)
            tracker.track_step("volume.get.call")
        finally:
            await self.drop()
            tracker.track_step("drop")
            tracker.track_e2e()
        return response

    async def perform_handshake(self, requests: list[Request], meta_requests: list[Request],
                                latency_tracker: LatencyTracker | None = None) -> None:
        tracker = latency_tracker or LatencyTracker("handshake")
        results = await self.storage_volume_ref.volume.handshake.call_one(self, meta_requests)
        tracker.track_step("volume.handshake.call")
        await self._post_handshake(results, requests)
        tracker.track_step("post_handshake")

    async def _post_handshake(self, handshake_results: list[Any], requests: list[Request]) -> None:
        pass

    async def _pre_put_hook(self, requests: list[Request]) -> None:
        pass

    async def _pre_get_hook(self, requests: list[Request]) -> None:
        pass

    async def _handle_storage_volume_response(self, requests: list[Request], response: Any) -> list[Any]:
        raise NotImplementedError()

    async def drop(self) -> None:
        pass

    # ---- volume side ----------------------------------------------------------------------------
    async def recv_handshake(self, ctx: "TransportContext", entries: list[tuple[Request, Any]]) -> list[Any]:
        raise NotImplementedError()

    async def handle_put_request(self, ctx: "TransportContext", entries: list[tuple[Request, Any]]) -> list[Any]:
        raise NotImplementedError()

    async def handle_get_request(self, ctx: "TransportContext", entries: list[tuple[Request, Any]]) -> None:
        raise NotImplementedError()


# ---------------------------------------------------------------------------------------------
# the landing-buffer put shared by the HBM transport and the host tier
# ---------------------------------------------------------------------------------------------
LANDING_TTL_S = 300.0


class LandingBuffers(TransportCache):
    """Volume side: landing buffers handed out by put handshakes, parked under (nonce, index) until
    the put stores them.  A put that fails between its handshake and its put never comes back for its
    buffers (the client's drop() cannot reach the volume), so every handshake first releases those
    parked for longer than ``LANDING_TTL_S``."""

    def __init__(self) -> None:
        self._parked: dict[tuple[str, int], tuple[float, torch.Tensor]] = {}

    def purge_stale(self) -> None:
        now = monotonic()
        for k in [k for k, (t, _) in self._parked.items() if now - t > LANDING_TTL_S]:
            del self._parked[k]

    def park(self, key: tuple[str, int], tensor: torch.Tensor) -> None:
        self._parked[key] = (monotonic(), tensor)

    def pop(self, key: tuple[str, int]) -> torch.Tensor | None:
        entry = self._parked.pop(key, None)
        return None if entry is None else entry[1]

    def clear(self) -> None:
        self._parked.clear()


@dataclass
class EntryContext:
    """Per-entry state carried inside the pickled buffer: where the tensor lives in volume memory,
    or the value that rides the RPC (objects, and tensors the transport cannot describe)."""

    descriptor: Any = None
    objects: Any = None
    use_rpc: bool = False


class LandingBufferTransport(TransportBuffer):
    """Two-phase put into volume memory.  At the handshake the volume hands out one landing buffer per
    tensor -- the stored tensor itself when shape, dtype and contiguity match and the transport can
    describe it (overwrite in place, reference storage_volume.py:161-207), else a new allocation --
    and parks it under (nonce, index).  The client copies into it (``_post_handshake``), and the put
    RPC pops it and stores it.  The per-buffer nonce keeps two clients putting the same key at once
    apart: each put stores the buffer its own handshake handed out.  Objects ride the RPC by value.

    A subclass supplies its volume memory (``_describe``, ``_allocate``) and its client-side copies
    (``_post_handshake``, ``_handle_storage_volume_response``)."""

    supports_batch_puts = True
    supports_batch_gets = True

    def __init__(self, storage_volume_ref: "StorageVolumeRef"):
        super().__init__(storage_volume_ref)
        self._nonce = os.urandom(8).hex()
        self._specs: list[tuple | None] = []  # put: (shape, dtype) of each tensor, None for an object
        self._contexts: list[EntryContext] = []

    # ---- volume memory: what each transport supplies ----------------------------------------------
    def _describe(self, ctx: TransportContext, tensor: torch.Tensor) -> Any | None:
        """Descriptor of a tensor (or view) in this transport's volume memory; None if it lives elsewhere."""
        raise NotImplementedError()

    def _allocate(self, ctx: TransportContext, shape: tuple, dtype: torch.dtype) -> tuple[torch.Tensor, Any]:
        """A new tensor in this transport's volume memory, with its descriptor."""
        raise NotImplementedError()

    # ---- client side ----------------------------------------------------------------------------
    def requires_handshake(self, requests: list[Request]) -> bool:
        return True

    async def perform_handshake(self, requests: list[Request], meta_requests: list[Request],
                                latency_tracker: LatencyTracker | None = None) -> None:
        self._specs = [None if r.is_object else (tuple(r.tensor_val.shape), r.tensor_val.dtype) for r in requests]
        await super().perform_handshake(requests, meta_requests, latency_tracker)

    async def drop(self) -> None:
        self._specs = []
        self._contexts = []

    # ---- volume side ----------------------------------------------------------------------------
    async def recv_handshake(self, ctx: TransportContext, entries: list[tuple[Request, Any]]) -> list[Any]:
        """Hand out where each tensor must be written."""
        parked = ctx.get(LandingBuffers)
        parked.purge_stale()
        out: list[Any] = []
        for idx, ((_, current), spec) in enumerate(zip(entries, self._specs, strict=True)):
            if spec is None:
                out.append(None)
                continue
            shape, dtype = spec
            desc = None
            if isinstance(current, torch.Tensor) and tuple(current.shape) == shape and current.dtype == dtype \
                    and current.is_contiguous():
                target, desc = current, self._describe(ctx, current)
            if desc is None:
                target, desc = self._allocate(ctx, shape, dtype)
            parked.park((self._nonce, idx), target)
            out.append(desc)
        return out

    async def handle_put_request(self, ctx: TransportContext, entries: list[tuple[Request, Any]]) -> list[Any]:
        """The stored values, aligned with ``entries``."""
        parked = ctx.get(LandingBuffers)
        results = []
        for idx, ((request, _), entry) in enumerate(zip(entries, self._contexts, strict=True)):
            if entry.use_rpc:
                results.append(entry.objects)
                continue
            target = parked.pop((self._nonce, idx))
            assert target is not None, f"No landing buffer for {request.key}: put without a matching handshake"
            results.append(target)
        return results

    async def handle_get_request(self, ctx: TransportContext, entries: list[tuple[Request, Any]]) -> None:
        self._contexts = []
        for request, data in entries:
            desc = None
            if not request.is_object and isinstance(data, torch.Tensor):
                desc = self._describe(ctx, data)
                if desc is None:
                    data = data.detach().cpu()  # stored by another tier: by value, on the host
            self._contexts.append(EntryContext(objects=data, use_rpc=True) if desc is None else EntryContext(descriptor=desc))

"""The transport plugin contract (reference torchstore/transport/buffers.py:20-361).

A ``TransportBuffer`` is created by the client for one (client, volume) pair, runs its client half
in the caller's process, is pickled into the volume RPCs and runs its volume half there.  The
lifecycle below is the reference's; ``transport/hbm.py`` is the implementation this repo ships.

PUT   requires_handshake? -> perform_handshake (volume: recv_handshake)
      -> _pre_put_hook -> RPC volume.put (volume: handle_put_request) -> _post_request_success
      -> drop (always)
GET   requires_handshake? -> perform_handshake -> _pre_get_hook
      -> RPC volume.get (volume: handle_get_request; the buffer object comes back)
      -> _handle_storage_volume_response -> _post_request_success -> drop (always)
"""

from __future__ import annotations

from abc import ABC, abstractmethod
from collections.abc import Iterable
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

    supports_inplace_resharding: bool = True
    supports_batch_puts: bool = False
    supports_batch_gets: bool = False
    supports_strided_inplace: bool = False  # in-place destinations may be non-contiguous views
    supports_fast_lane: bool = False        # has a ``record`` flag and ``take_recorded`` (fast_lane.py)

    def __init__(self, storage_volume_ref: "StorageVolumeRef"):
        self.storage_volume_ref = storage_volume_ref
        self._volume_epoch = None  # the volume's layout epoch after the last put (storage_volume.py)

    # ---- client side ----------------------------------------------------------------------------
    def requires_handshake(self, requests: list[Request]) -> bool:
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
            await self._post_request_success()
            tracker.track_step("_post_request_success")
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
            if self.requires_handshake(requests):
                await self.perform_handshake(requests, meta, tracker)
            await self._pre_get_hook(requests)
            tracker.track_step("_pre_get_hook")
            returned = await self.storage_volume_ref.volume.get.call_one(self, meta)
            response = await self._handle_storage_volume_response(requests, returned)
            tracker.track_step("volume.get.call")
            await self._post_request_success()
            tracker.track_step("_post_request_success")
        finally:
            await self.drop()
            tracker.track_step("drop")
            tracker.track_e2e()
        return response

    async def perform_handshake(self, requests: list[Request], meta_requests: list[Request],
                                latency_tracker: LatencyTracker | None = None) -> None:
        """Default: one RPC.  Multi-stage transports override this."""
        tracker = latency_tracker or LatencyTracker("handshake")
        await self._pre_handshake()
        tracker.track_step("pre_handshake")
        results = await self.storage_volume_ref.volume.handshake.call_one(self, meta_requests)
        tracker.track_step("volume.handshake.call")
        await self._post_handshake(results, requests)
        tracker.track_step("post_handshake")

    async def _pre_handshake(self) -> None:
        pass

    async def _post_handshake(self, handshake_results: list[Any], requests: list[Request]) -> None:
        pass

    async def _post_request_success(self) -> None:
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

    # ---- helpers --------------------------------------------------------------------------------
    def _assert_valid_tensor(self, tensor: torch.Tensor, dtype: torch.dtype, shape: torch.Size,
                             must_be_contiguous: bool = True) -> None:
        assert isinstance(tensor, torch.Tensor)
        assert tensor.dtype == dtype, f"{tensor.dtype} != {dtype}"
        assert tensor.shape == shape, f"{tensor.shape} != {shape}"
        assert not must_be_contiguous or tensor.is_contiguous()

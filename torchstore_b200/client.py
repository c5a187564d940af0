"""LocalClient: the in-process half of the store (reference torchstore/client.py:29-496).

Builds Requests, picks the volume (strategy), drives the transport, and plans reshard fetches:
every stored rectangle that intersects the wanted rectangle becomes one sub-request whose
destination is a *view* of the caller's tensor, so a whole ``get_batch`` turns into one
copy_rects launch per (volume, destination GPU) with no assemble step.  When the caller gives no
destination the bounding box is gathered on the GPU first and moved to the host once.
"""

from __future__ import annotations

import asyncio
from collections import defaultdict
from logging import getLogger
from typing import Any

import torch
from torch.distributed.tensor import DTensor

from torchstore_b200 import _native
from torchstore_b200.controller import ObjectType
from torchstore_b200.fast_lane import FastLane, Recording, signature
from torchstore_b200.launch import staging_copy, wait_copy_stream
from torchstore_b200.logging import LatencyTracker
from torchstore_b200.strategy import TorchStoreStrategy
from torchstore_b200.transport import Request, TensorSlice, create_transport_buffer
from torchstore_b200.transport.hbm import get_result_device
from torchstore_b200.utils import (
    assemble_tensor,
    get_destination_region,
    get_destination_view,
    get_slice_intersection,
    get_target_tensor_shape_and_offset,
    tensors_overlap_in_memory,
)

logger = getLogger(__name__)


class GatherTarget:
    """Bounding-box buffer a sharded key is gathered into when the caller gave no destination.
    Allocated lazily on the GPU by the transport once the stored dtype is known; every
    sub-request of the key (possibly from several volumes) lands in a view of it."""

    def __init__(self, shape, origin) -> None:
        self.shape = tuple(shape)
        self.origin = tuple(origin)
        self.tensor: torch.Tensor | None = None

    def view_for(self, fetch: TensorSlice, dtype: torch.dtype, device) -> torch.Tensor:
        if self.tensor is None:
            self.tensor = torch.empty(self.shape, dtype=dtype, device=device)
        idx = tuple(slice(o - b, o - b + s) for o, b, s in zip(fetch.offsets, self.origin, fetch.local_shape))
        return self.tensor[idx]


class PendingPut:
    """Returned by ``put_batch(..., wait=False)``: the copy is running on the side stream; awaiting
    the object completes the put (data committed and readable by any client).  The caller must not
    overwrite the source tensors before that."""

    def __init__(self, finish=None) -> None:
        self._finish = finish
        self.done = finish is None

    def __await__(self):
        return self.wait().__await__()

    async def wait(self) -> None:
        if not self.done:
            await self._finish()
            self.done = True


class LocalClient:
    def __init__(self, controller, strategy) -> None:
        self._controller = controller
        self.strategy: TorchStoreStrategy = strategy
        self.fast_lane = FastLane(controller, strategy)

    async def _locate_volumes(self, keys: list[str]):
        try:
            return await self._controller.locate_volumes.call_one(keys)
        except Exception as e:
            raise KeyError(str(e)) from e

    # ---- put ------------------------------------------------------------------------------------
    @torch.no_grad
    async def put(self, key: str, value: torch.Tensor | Any):
        tracker = LatencyTracker(f"put:{key}")
        await self.put_batch({key: value})
        tracker.track_e2e()

    @torch.no_grad
    async def put_batch(self, entries: dict[str, torch.Tensor | Any], wait: bool = True):
        """``wait=False`` (extension): return a :class:`PendingPut` as soon as the copy has been
        enqueued on the side stream, so it overlaps the caller's compute; ``await`` it to complete
        the put.  Only a batch served by the fast lane (put before, nothing moved) can return early;
        a first put completes inline and returns an already-finished PendingPut."""
        assert isinstance(entries, dict) and entries, "put_batch requires a non-empty dict"
        tracker = LatencyTracker("put_batch")
        requests = [
            Request.from_any(k, v) if isinstance(v, (torch.Tensor, DTensor)) else Request.from_objects(k, v)
            for k, v in entries.items()
        ]
        volume_ref = self.strategy.select_storage_volume()
        transport = create_transport_buffer(volume_ref)
        tracker.track_step("create transport buffer")
        sig = signature(requests, volume_ref.volume_id) if transport.supports_fast_lane else None
        rec = None
        if sig is not None:
            replay = await self.fast_lane.replay_put(sig)
            if replay is not None:  # keys overwritten in place: the index is already right, no notify
                if wait:
                    await replay.wait()
                tracker.track_e2e()
                return None if wait else PendingPut(replay.wait)
            rec = Recording(sig)
            rec.attach([transport])
        ok = False
        try:
            await transport.put_to_storage_volume(requests)
            tracker.track_step("put_to_storage_volume")
            await self._controller.notify_put_batch.call([r.meta_only() for r in requests], volume_ref.volume_id)
            tracker.track_step("notify_put_batch")
            ok = True
        finally:
            if rec is not None:
                self.fast_lane.commit(rec, ok)
        tracker.track_e2e()
        return None if wait else PendingPut()

    # ---- get ------------------------------------------------------------------------------------
    @torch.no_grad
    async def get(self, key: str, inplace_tensor: torch.Tensor | DTensor | None = None,
                  tensor_slice_spec: TensorSlice | None = None):
        logger.debug("Fetching %s", key)
        tracker = LatencyTracker(f"get:{key}")
        request = Request.from_any(key, inplace_tensor, tensor_slice_spec)
        results = await self._fetch([request])
        tracker.track_step("fetch")
        out = self._apply_inplace(results[key], inplace_tensor, request)
        tracker.track_e2e()
        return out

    @torch.no_grad
    async def get_batch(self, keys: list[str] | dict[str, torch.Tensor | DTensor | None]) -> dict[str, Any]:
        tracker = LatencyTracker("get_batch")
        if not keys:
            raise ValueError("get_batch requires a non-empty dict or list")
        inplace: dict = {}
        if isinstance(keys, dict):
            inplace = keys
        elif isinstance(keys, list):
            if len(keys) != len(set(keys)):
                raise ValueError("get_batch keys must be unique")
        else:
            raise TypeError(f"get_batch expects list[str] or dict, got {type(keys)}")
        requests = [Request.from_any(k, inplace.get(k)) for k in keys]
        sig = signature(requests)
        rec = None
        if sig is not None:
            replay = await self.fast_lane.replay_get(sig)
            if replay is not None:
                tracker.track_e2e()
                return replay
            rec = await self.fast_lane.record_get(sig)
        results = final = None
        try:
            results = await self._fetch(requests, rec)
            tracker.track_step("fetch")
            final = {r.key: self._apply_inplace(results[r.key], inplace.get(r.key), r) for r in requests}
        finally:
            if rec is not None:
                self.fast_lane.finish_get(rec, requests, results, final)
        tracker.track_e2e()
        return final

    def close_sessions(self) -> None:
        self.fast_lane.clear()

    def _apply_inplace(self, fetched: Any, inplace_tensor, request: Request) -> Any:
        """Always hand back the caller's object; copy only if the fetch could not land in place."""
        if inplace_tensor is not None and fetched.data_ptr() != request.tensor_val.data_ptr():
            request.tensor_val.copy_(fetched)
            return inplace_tensor
        return inplace_tensor if inplace_tensor is not None else fetched

    async def _fetch(self, requests: list[Request], recording: Recording | None = None) -> dict[str, Any]:
        volume_maps = await self._locate_volumes([r.key for r in requests])
        volume_ids = {vid for vm in volume_maps.values() for vid in vm}
        transports = {vid: create_transport_buffer(self.strategy.get_storage_volume(vid)) for vid in volume_ids}
        volume_requests, whole_keys, gathers = self._build_volume_requests(requests, volume_maps, transports)
        if recording is not None:
            recording.attach([transports[v] for v in volume_requests])
        pairs = await self._fetch_results(volume_requests, transports)
        return await self._assemble_results(requests, pairs, whole_keys, gathers)

    def _build_volume_requests(self, requests, volume_maps, transports):
        """Per-key requests -> per-volume sub-request lists.

        Returns (volume_requests, whole_keys, gathers): whole_keys are stored as one OBJECT/TENSOR;
        gathers maps a key fetched without a destination to the GPU bounding-box buffer its
        rectangles are gathered into."""
        volume_requests: dict[str, list[Request]] = defaultdict(list)
        whole_keys: set[str] = set()
        gathers: dict[str, torch.Tensor] = {}
        for request in requests:
            volume_map = volume_maps[request.key]
            strided_ok = all(transports[v].supports_strided_inplace for v in volume_map)
            use_inplace = request.tensor_val is not None and (strided_ok or request.tensor_val.is_contiguous())
            sharded: list[tuple[str, TensorSlice]] = []
            for volume_id, info in volume_map.items():
                if info.object_type == ObjectType.OBJECT:
                    volume_requests[volume_id].append(Request(key=request.key, is_object=True))
                    whole_keys.add(request.key)
                    break
                if info.object_type == ObjectType.TENSOR:
                    volume_requests[volume_id].append(request)
                    whole_keys.add(request.key)
                    break
                for stored in info.tensor_slices:
                    fetch = stored
                    if request.tensor_slice is not None:
                        fetch = get_slice_intersection(stored, request.tensor_slice)
                        if fetch is None:
                            continue
                    sharded.append((volume_id, fetch))
            if not sharded:
                continue
            # replicated shards: every region once (the reference re-fetches duplicates, client.py:295-297)
            seen, unique = set(), []
            for volume_id, fetch in sharded:
                region = (fetch.offsets, fetch.local_shape)
                if region not in seen:
                    seen.add(region)
                    unique.append((volume_id, fetch))
            gather = None
            if request.tensor_val is None and strided_ok:
                shape, origin = get_target_tensor_shape_and_offset(
                    [f.local_shape for _, f in unique], [f.offsets for _, f in unique]
                )
                gather = gathers[request.key] = GatherTarget(shape, origin)
            for volume_id, fetch in unique:
                sub = Request.from_tensor_slice(request.key, fetch)
                if use_inplace:
                    pick = get_destination_region if strided_ok else get_destination_view
                    view = pick(request.tensor_val, request.tensor_slice, fetch)
                    if view is not None:
                        sub.tensor_val = view
                elif gather is not None:
                    sub._gather = gather  # client-only: stripped by meta_only()
                volume_requests[volume_id].append(sub)
        return dict(volume_requests), whole_keys, gathers

    async def _fetch_results(self, volume_requests, transports):
        async def one(volume_id, subs):
            results = await transports[volume_id].get_from_storage_volume(subs)
            return list(zip(subs, results, strict=True))

        per_volume = await asyncio.gather(*[one(v, s) for v, s in volume_requests.items()])
        return [pair for pairs in per_volume for pair in pairs]

    async def _assemble_results(self, requests, fetch_pairs, whole_keys, gathers) -> dict[str, Any]:
        final: dict[str, Any] = {}
        parts: dict[str, list] = defaultdict(list)
        for sub, result in fetch_pairs:
            if sub.key in whole_keys:
                final[sub.key] = result
            else:
                parts[sub.key].append((result, sub.tensor_slice))
        by_key = {r.key: r for r in requests}
        for key, plist in parts.items():
            request = by_key[key]
            if request.tensor_val is not None and tensors_overlap_in_memory(plist, request.tensor_val):
                final[key] = request.tensor_val
            elif key in gathers and gathers[key].tensor is not None and tensors_overlap_in_memory(plist, gathers[key].tensor):
                final[key] = await self._to_result_device(gathers[key].tensor)
            else:
                tensors = [t for t, _ in plist]
                final[key] = assemble_tensor(tensors, [s.offsets for _, s in plist], device=tensors[0].device)
            if request.tensor_slice is not None and final[key] is not request.tensor_val:
                assert final[key].shape == request.tensor_slice.local_shape
        for r in requests:
            if r.key not in final:
                raise RuntimeError(
                    f"No results found for key '{r.key}'. If this key contains tensor slices, no stored slices "
                    "intersect with the requested slice."
                )
        return final

    async def _to_result_device(self, gathered: torch.Tensor) -> torch.Tensor:
        if get_result_device() == "cuda" or not gathered.is_cuda:
            return gathered
        host = torch.empty(gathered.shape, dtype=gathered.dtype)
        dev = gathered.device.index
        staging_copy(dev, host.data_ptr(), gathered.data_ptr(), gathered.numel() * gathered.element_size(), _native.TSB_D2H)
        await wait_copy_stream(dev)
        return host

    # ---- misc -----------------------------------------------------------------------------------
    async def keys(self, prefix: str | None = None) -> list[str]:
        return await self._controller.keys.call_one(prefix)

    async def delete(self, key: str) -> None:
        tracker = LatencyTracker(f"delete:{key}")
        volume_map = (await self._controller.locate_volumes.call_one([key]))[key]

        async def one(volume_id: str):
            ref = self.strategy.get_storage_volume(volume_id)
            # notify first so the index never points at a volume that is deleting
            await self._controller.notify_delete.call_one(key, volume_id)
            await ref.volume.delete.call(key)

        await asyncio.gather(*[one(v) for v in volume_map])
        self.strategy.transport_context.delete(key)
        tracker.track_e2e()

    async def delete_batch(self, keys: list[str]) -> None:
        if not isinstance(keys, list):
            raise TypeError(f"delete_batch expects list[str], got {type(keys)}")
        unique = list(dict.fromkeys(keys))
        if not unique:
            return
        tracker = LatencyTracker("delete_batch")
        volume_maps = await self._controller.locate_volumes.call_one(unique, missing_ok=True,
                                                                     require_fully_committed=False)
        tracker.track_step("locate_volumes")
        by_volume: dict[str, list[str]] = defaultdict(list)
        for key, vm in volume_maps.items():
            for volume_id in vm:
                by_volume[volume_id].append(key)
        if by_volume:
            await self._controller.notify_delete_batch.call_one(dict(by_volume))
            tracker.track_step("notify_delete_batch")

        async def one(volume_id: str, vkeys: list[str]):
            await self.strategy.get_storage_volume(volume_id).volume.delete_batch.call(vkeys)

        await asyncio.gather(*[one(v, k) for v, k in by_volume.items()])
        tracker.track_step("volume.delete_batch")
        self.strategy.transport_context.delete(unique)
        tracker.track_step("transport_context.delete")
        tracker.track_e2e()

    async def exists(self, key: str) -> bool:
        logger.debug("Checking existence of %s", key)
        try:
            await self._controller.locate_volumes.call_one([key])
            return True
        except Exception as e:
            if "KeyError" in str(e) or "Unable to locate" in str(e):
                return False
            raise

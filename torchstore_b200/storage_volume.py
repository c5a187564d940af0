"""Storage volume: a key/value store whose tensors live in HBM arenas on one GPU of the box.

Counterpart of the reference's ``torchstore/storage_volume.py`` (StorageVolume :25-99,
InMemoryStore :146-407) with one change of substance: tensor bytes are kept in device memory
carved from ``tsb_arena`` slabs (one cudaMalloc each, exportable over CUDA IPC) instead of POSIX
shared-memory segments, so a reader on any GPU pulls them over NVLink with the copy_rects kernel
and never crosses PCIe.  Objects are kept by value.

Stored forms (same as the reference's ``kv``):
    kv[key] = tensor                                   plain tensor
    kv[key] = {"obj": value}                           python object
    kv[key] = {coords: {"slice": TensorSlice, "tensor": tensor}, ...}   one entry per stored shard
"""

from __future__ import annotations

import os
import socket
from logging import getLogger
from typing import Any

import torch

from torchstore_b200.rpc import Actor, endpoint
from torchstore_b200.transport.buffers import TransportBuffer, TransportContext
from torchstore_b200.transport.types import Request, TensorSlice
from torchstore_b200.utils import get_slice_intersection

logger = getLogger(__name__)

FULL_TENSOR = "full_tensor"


# ---------------------------------------------------------------------------------------------
# the actor
# ---------------------------------------------------------------------------------------------
class StorageVolume(Actor):
    """Remote half of the store: receives handshake/put/get/delete requests for one volume."""

    actor_name: str = "StorageVolumes"

    def __init__(self, id_func, device: int | None = None) -> None:
        self.volume_id: str = id_func()
        self.store: StorageImpl = InMemoryStore(device=_pick_device(self.volume_id, device))

    @endpoint
    async def get_id(self) -> tuple[str, str]:
        return (self.volume_id, os.environ.get("HOSTNAME", socket.gethostname()))

    @endpoint
    async def handshake(self, transport_buffer: TransportBuffer, requests: list[Request]) -> list[Any]:
        return await self.store.handshake(transport_buffer, requests)

    @endpoint
    async def put(self, transport_buffer: TransportBuffer, requests: list[Request]) -> int:
        """Returns the volume's layout epoch after the put (see InMemoryStore.epoch)."""
        await self.store.put(transport_buffer, requests)
        return self.store.epoch

    @endpoint
    async def epoch(self) -> int:
        return self.store.epoch

    @endpoint
    async def attach_epoch_board(self, name: str, slot: int) -> bool:
        """Mirror this volume's layout epoch into slot `slot` of the controller's epoch board."""
        return self.store.attach_epoch_board(name, slot)

    @endpoint
    async def get(self, transport_buffer: TransportBuffer, requests: list[Request]) -> TransportBuffer:
        return await self.store.get(transport_buffer, requests)

    @endpoint
    async def get_meta(self, requests: list[Request]) -> list[tuple[torch.Size, torch.dtype] | str]:
        return await self.store.get_meta(requests)

    @endpoint
    async def delete(self, key: str) -> None:
        await self.store.delete(key)
        self.store.transport_context.delete(key)

    @endpoint
    async def delete_batch(self, keys: list[str]) -> None:
        await self.store.delete_batch(keys)
        self.store.transport_context.delete(keys)

    @endpoint
    async def reset(self) -> None:
        self.store.reset()

    @endpoint
    async def stats(self) -> dict:
        return self.store.stats()


def _pick_device(volume_id: str, device: int | None) -> int | None:
    if not torch.cuda.is_available():
        return None
    n = torch.cuda.device_count()
    if device is not None:
        return device % n
    local = os.environ.get("LOCAL_RANK")
    if local is not None and os.environ.get("TORCHSTORE_B200_VOLUME_DEVICE_FROM_ID", "0") != "1":
        return int(local) % n
    return int(volume_id) % n if volume_id.isdigit() else 0


class StorageImpl:
    def __init__(self) -> None:
        self.transport_context = TransportContext()
        self.epoch = 0
        self._board = None
        self._board_slot = 0

    def _bump(self) -> None:
        self.epoch += 1
        if self._board is not None:
            self._board.write(self._board_slot, self.epoch)

    def attach_epoch_board(self, name: str, slot: int) -> bool:
        from torchstore_b200 import epoch_board

        board = epoch_board.attached(name)
        if board is None:
            return False
        self._board, self._board_slot, self._board_name = board, slot, name
        board.write(slot, self.epoch)
        return True

    def detach_epoch_board(self) -> None:
        if self._board is not None:
            from torchstore_b200 import epoch_board

            self._board = None
            epoch_board.forget(getattr(self, "_board_name", None))

    async def put(self, transport_buffer: TransportBuffer, requests: list[Request]) -> None:
        raise NotImplementedError()

    async def get(self, transport_buffer: TransportBuffer, requests: list[Request]) -> TransportBuffer:
        raise NotImplementedError()

    async def get_meta(self, requests: list[Request]):
        raise NotImplementedError()

    async def delete(self, key: str) -> None:
        raise NotImplementedError()

    async def delete_batch(self, keys: list[str]) -> None:
        raise NotImplementedError()

    async def handshake(self, transport_buffer: TransportBuffer, requests: list[Request]) -> list[Any]:
        raise NotImplementedError()


class InMemoryStore(StorageImpl):
    """Dict store over HBM-resident tensors."""

    def __init__(self, device: int | None = None) -> None:
        super().__init__()
        self.kv: dict[str, Any] = {}
        self.device = device
        # layout epoch: bumped whenever a key starts pointing at OTHER memory (new key, reallocation,
        # delete, reset) -- never by an in-place overwrite.  A client's cached put/get plan (device
        # pointers into this volume's arenas) is valid exactly while the epoch it was built under lasts.
        self._configure_transport()

    def _configure_transport(self) -> None:
        # the HBM transport's volume half allocates stored tensors from this volume's arenas
        from torchstore_b200.transport.hbm import HbmVolumeCache

        self.transport_context.get(HbmVolumeCache).configure(self.device)

    def stats(self) -> dict:
        from torchstore_b200.transport.hbm import HbmVolumeCache

        out = {"keys": len(self.kv), "device": self.device}
        out.update(self.transport_context.get(HbmVolumeCache).stats())
        return out

    # -- existing-entry lookup (in-place overwrite support) ------------------------------------------
    def _extract_existing(self, request: Request) -> torch.Tensor | None:
        current = self.kv.get(request.key)
        if current is None:
            return None
        if isinstance(current, torch.Tensor):
            assert request.tensor_slice is None, (
                "Existing data is a regular tensor but incoming request has tensor_slice (DTensor)"
            )
            return current
        if isinstance(current, dict):
            if "obj" in current:
                assert request.is_object, "Existing data is an object but request.is_object is False"
                return None
            assert request.tensor_slice is not None, (
                "Existing data is DTensor shards but incoming request has no tensor_slice"
            )
            shard = current.get(request.tensor_slice.coordinates)
            return shard["tensor"] if shard is not None and "tensor" in shard else None
        raise AssertionError(f"Unexpected current_object type: {type(current)}")

    async def handshake(self, transport_buffer: TransportBuffer, requests: list[Request]) -> list[Any]:
        pairs = [(r, self._extract_existing(r)) for r in requests]
        return await transport_buffer.recv_handshake(self.transport_context, pairs)

    # -- put ------------------------------------------------------------------------------------
    async def put(self, transport_buffer: TransportBuffer, requests: list[Request]) -> None:
        entries = [(r, self._extract_existing(r)) for r in requests]
        results = await transport_buffer.handle_put_request(self.transport_context, entries)
        for request, data in zip(requests, results, strict=True):
            self._store(request, data)

    def _store(self, request: Request, data: Any) -> None:
        if request.is_object:
            if not isinstance(self.kv.get(request.key), dict) or "obj" not in self.kv[request.key]:
                self._bump()
            self.kv[request.key] = {"obj": data}
        elif request.tensor_slice is not None:
            shards = self.kv.setdefault(request.key, {})
            old = shards.get(request.tensor_slice.coordinates)
            if old is None or old.get("tensor") is not data or old.get("slice") != request.tensor_slice:
                self._bump()
            shards[request.tensor_slice.coordinates] = {"slice": request.tensor_slice, "tensor": data}
        else:
            if self.kv.get(request.key) is not data:
                self._bump()
            self.kv[request.key] = data

    # -- get ------------------------------------------------------------------------------------
    @staticmethod
    def _box(tensor: torch.Tensor, offsets, shape) -> torch.Tensor:
        return tensor[tuple(slice(o, o + s) for o, s in zip(offsets, shape))]

    def _get_sharded_tensor(self, request: Request) -> torch.Tensor | None:
        """View of the first stored shard that fully contains the requested rectangle."""
        want = request.tensor_slice
        for shard in self.kv[request.key].values():
            stored: TensorSlice = shard["slice"]
            inter = get_slice_intersection(stored, want)
            if inter is None or inter.local_shape != want.local_shape or inter.offsets != want.offsets:
                continue
            local = [inter.offsets[d] - stored.offsets[d] for d in range(len(inter.offsets))]
            return self._box(shard["tensor"], local, inter.local_shape)
        return None

    def _get_data(self, request: Request):
        val = self.kv[request.key]
        if isinstance(val, dict) and "obj" in val:
            return val["obj"]
        if isinstance(val, torch.Tensor):
            if request.tensor_slice is None:
                return val
            return self._box(val, request.tensor_slice.offsets, request.tensor_slice.local_shape)
        if request.tensor_slice is None:
            raise RuntimeError(f"Key '{request.key}' contains sharded tensor but no tensor_slice was requested")
        view = self._get_sharded_tensor(request)
        if view is None:
            raise RuntimeError(f"Tensor slice {request.tensor_slice} not found in any stored shards for {request.key}")
        return view

    async def get(self, transport_buffer: TransportBuffer, requests: list[Request]) -> TransportBuffer:
        entries = []
        for request in requests:
            if request.key not in self.kv:
                raise KeyError(f"Key '{request.key}' not found. {list(self.kv.keys())=}")
            entries.append((request, self._get_data(request)))
        # the layout epoch the client's fast lane files a get's plans under (StorageVolume.put returns it)
        transport_buffer._volume_epoch = self.epoch
        await transport_buffer.handle_get_request(self.transport_context, entries)
        return transport_buffer

    async def get_meta(self, requests: list[Request]):
        return [self._get_meta(r) for r in requests]

    def _get_meta(self, request: Request):
        if request.key not in self.kv:
            raise KeyError(f"Key '{request.key}' not found. {list(self.kv.keys())=}")
        val = self.kv[request.key]
        if isinstance(val, torch.Tensor):
            return val.shape, val.dtype
        assert isinstance(val, dict)
        if "obj" in val:
            return "obj"
        if request.tensor_slice is not None:
            view = self._get_sharded_tensor(request)
            if view is not None:
                return view.shape, view.dtype
            raise KeyError(f"Could not find shard slice with {request.tensor_slice=}  Slices:{val}")
        raise RuntimeError(f"Unknown type for {request.key} type={type(val)} {val=}")

    # -- delete / reset ----------------------------------------------------------------------------
    async def delete(self, key: str) -> None:
        if key not in self.kv:
            raise KeyError(f"Key '{key}' not found. {list(self.kv.keys())=}")
        del self.kv[key]
        self._bump()

    async def delete_batch(self, keys: list[str]) -> None:
        for key in set(keys):
            if self.kv.pop(key, None) is not None:
                self._bump()

    def reset(self) -> None:
        self.kv = {}
        self._bump()
        self._board = None  # the controller that published the board is tearing the store down
        self.transport_context.clear()
        self._configure_transport()

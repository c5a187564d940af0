"""By-value transport: the data rides the actor RPC itself (reference
``MonarchRPCTransportBuffer``, transport/monarch_rpc.py:26-90).

Selected ONLY by ``TransportType.MonarchRPC`` -- never automatically.  It exists for the cases the
reference uses it for: tiny control tensors and objects between processes that share nothing (no
NVLink peer mapping, no common /dev/shm).  The buffer carries the payload as a member, so whatever
actor layer delivers the call (this build: ``rpc.py``; Monarch endpoints behave the same, the class
only relies on the ``TransportBuffer`` hooks) serialises it with the buffer.  GPU tensors are staged
to the host first, exactly like torch's pickling of a CUDA tensor would; bandwidth-sized keys belong
on the NVLink/HBM transport.
"""

from __future__ import annotations

from typing import TYPE_CHECKING, Any

import torch

from torchstore_b200.transport.buffers import TransportBuffer
from torchstore_b200.transport.types import Request

if TYPE_CHECKING:
    from torchstore_b200.strategy import StorageVolumeRef
    from torchstore_b200.transport.buffers import TransportContext


class ActorRpcTransportBuffer(TransportBuffer):
    supports_batch_puts = True
    supports_batch_gets = True
    supports_strided_inplace = True  # Tensor.copy_ into any view

    def __init__(self, storage_volume_ref: "StorageVolumeRef"):
        super().__init__(storage_volume_ref)
        self.data: list[Any] = []              # payload, aligned with the requests of the call
        self._inplace: list[torch.Tensor | None] = []

    def __getstate__(self) -> dict[str, Any]:
        state = super().__getstate__()
        state["_inplace"] = []                 # destinations never travel
        return state

    async def _pre_put_hook(self, requests: list[Request]) -> None:
        self.data = [r.objects if r.is_object else r.tensor_val.detach().cpu().contiguous() for r in requests]

    async def _pre_get_hook(self, requests: list[Request]) -> None:
        self._inplace = [r.tensor_val for r in requests]

    async def handle_put_request(self, ctx: "TransportContext", entries: list[tuple[Request, Any]]) -> list[Any]:
        assert len(entries) == len(self.data)
        out = []
        for (request, current), value in zip(entries, self.data):
            if isinstance(value, torch.Tensor) and isinstance(current, torch.Tensor) and not current.is_cuda \
                    and current.shape == value.shape and current.dtype == value.dtype:
                current.copy_(value)           # overwrite in place (storage_volume.py:161-207)
                out.append(current)
            else:
                out.append(value)
        return out

    async def handle_get_request(self, ctx: "TransportContext", entries: list[tuple[Request, Any]]) -> None:
        self.data = [d.detach().cpu().contiguous() if isinstance(d, torch.Tensor) else d for _, d in entries]

    async def _handle_storage_volume_response(self, requests: list[Request], transport_buffer: "TransportBuffer") -> list[Any]:
        results = []
        for request, dest, value in zip(requests, self._inplace, transport_buffer.data, strict=True):
            gather = getattr(request, "_gather", None)
            if dest is None and gather is not None and isinstance(value, torch.Tensor):
                dest = gather.view_for(request.tensor_slice, value.dtype, torch.device("cpu"))
            if dest is not None and isinstance(value, torch.Tensor):
                dest.copy_(value)              # converting, any device, any strides
                results.append(dest)
            else:
                results.append(value)
        return results

    async def drop(self) -> None:
        self.data = []
        self._inplace = []

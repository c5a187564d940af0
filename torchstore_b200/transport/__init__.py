"""Transport registry.  This build ships two data tiers: the NVLink/HBM transport
(``transport/hbm.py``, the default wherever a CUDA device exists) and the host tier
(``transport/host.py``: POSIX shm volumes for CPU clients and GPU-less boxes, the reference's
``TransportType.SharedMemory``), plus the by-value ``TransportType.MonarchRPC`` transport
(``transport/actor_rpc.py``) for explicit use.  The enum keeps the reference's member names
(transport/__init__.py:34-42) so existing ``Strategy(default_transport_type=...)`` call sites still
import; selecting a transport that is not part of this build fails loudly instead of falling back."""

from __future__ import annotations

from enum import Enum, auto
from typing import TYPE_CHECKING

from torchstore_b200.transport.buffers import TransportBuffer
from torchstore_b200.transport.types import Request, TensorSlice

if TYPE_CHECKING:
    from torchstore_b200.strategy import StorageVolumeRef


class TransportType(Enum):
    Unset = auto()  # resolved lazily: NVLink on this build
    MonarchRPC = auto()
    MonarchRDMA = auto()
    TorchComms = auto()
    TorchCommsRDMA = TorchComms
    Gloo = auto()
    SharedMemory = auto()
    NVLink = auto()  # HBM arena volumes + P2P copy_rects over NVSwitch (this repo)


def get_available_transport(storage_volume_ref: "StorageVolumeRef") -> TransportType:
    """NVLink wherever this process can see a CUDA device; the host tier only in a process with no
    GPU at all (reference auto-selection: strategy.py:45-63)."""
    import torch

    return TransportType.NVLink if torch.cuda.is_available() else TransportType.SharedMemory


def create_transport_buffer(storage_volume_ref: "StorageVolumeRef") -> TransportBuffer:
    transport_type = storage_volume_ref.default_transport_type
    if transport_type == TransportType.Unset:
        transport_type = get_available_transport(storage_volume_ref)
    if transport_type == TransportType.NVLink:
        from torchstore_b200.transport.hbm import HbmTransportBuffer

        return HbmTransportBuffer(storage_volume_ref)
    if transport_type == TransportType.SharedMemory:
        from torchstore_b200.transport.host import HostShmTransportBuffer

        return HostShmTransportBuffer(storage_volume_ref)
    if transport_type == TransportType.MonarchRPC:
        # by value through the actor RPC: explicit choice only, never auto-selected
        from torchstore_b200.transport.actor_rpc import ActorRpcTransportBuffer

        return ActorRpcTransportBuffer(storage_volume_ref)
    raise RuntimeError(
        f"transport {transport_type.name} is not part of the torchstore_b200 build; use TransportType.NVLink (HBM volumes), "
        "TransportType.SharedMemory (host tier), TransportType.MonarchRPC (by value through the actor RPC) or leave "
        "default_transport_type unset"
    )


__all__ = ["Request", "TensorSlice", "TransportType", "create_transport_buffer", "get_available_transport"]

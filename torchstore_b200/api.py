"""Module-level coroutines: the user-facing API (reference torchstore/api.py:33-438).

Signatures are the reference's.  ``initialize`` builds the single-box control plane in THIS
process (controller + ``num_storage_volumes`` HBM volumes); under torchrun use
``torchstore_b200.initialize_spmd`` so every rank hosts its own volume.
"""

from __future__ import annotations

from typing import TYPE_CHECKING, Any

import torch
from torch.distributed.tensor import DTensor

import torchstore_b200.state_dict_utils as state_dict_utils
from torchstore_b200 import rpc
from torchstore_b200 import strategy as strategy_mod
from torchstore_b200.client import LocalClient
from torchstore_b200.controller import Controller
from torchstore_b200.storage_volume import StorageVolume
from torchstore_b200.strategy import ControllerStorageVolumes, TorchStoreStrategy
from torchstore_b200.transport.types import TensorSlice

if TYPE_CHECKING:
    from torchstore_b200.spmd import _SPMDSession

DEFAULT_TORCHSTORE_NAME: str = "torchstore"

_local_clent_map: dict[str, LocalClient] = {}
_spmd_state_map: dict[str, "_SPMDSession"] = {}
_controllers: dict[str, Any] = {}  # store name -> controller ref (single-process stores)
_owned_actors: dict[str, list[str]] = {}


def _spawn_volumes(num: int, strategy: TorchStoreStrategy, store_name: str):
    """Volumes of a single-process store: volume i is numbered by the strategy as if spawned on
    rank i and keeps its tensors on GPU i % device_count."""
    members = []
    names = _owned_actors.setdefault(store_name, [])
    for i in range(num):
        strategy_mod._spawn_rank[0] = i
        vol = StorageVolume(id_func=strategy.get_volume_id, device=i if torch.cuda.is_available() else None)
        name = f"{store_name}/volume/{i}"
        names.append(name)
        members.append(({"gpus": i}, rpc.register_actor(name, vol)))
    strategy_mod._spawn_rank[0] = 0
    return members


async def initialize(num_storage_volumes: int = 1, strategy: TorchStoreStrategy | None = None,
                     store_name: str = DEFAULT_TORCHSTORE_NAME, mesh=None) -> None:
    """Set up volumes and controller; must run before any put/get.

    ``mesh`` (a Monarch ProcMesh in the reference) is accepted for signature compatibility and
    ignored: on one box volumes are HBM arenas of this process' GPUs."""
    if num_storage_volumes == 1 and strategy is None:
        strategy = ControllerStorageVolumes()
    elif strategy is None:
        raise RuntimeError("Must specify controller strategy if num_storage_volumes > 1")
    if store_name in _controllers or store_name in _spmd_state_map:
        # refuse BEFORE spawning: registering fresh volumes under the live store's actor names would
        # replace its data (the reference leaves an initialised store intact, controller.py:118-121)
        raise RuntimeError(f"TorchStore '{store_name}' is already initialized in this process; call shutdown() first")
    members = _spawn_volumes(num_storage_volumes, strategy, store_name)
    if isinstance(strategy, ControllerStorageVolumes):
        storage_volumes = members[0][1]
    else:
        storage_volumes = rpc.ActorMesh(members)
    controller = await _controller(store_name, create=True)
    await controller.init.call(strategy=strategy, num_storage_volumes=num_storage_volumes,
                               storage_volumes=storage_volumes)


async def shutdown(store_name: str = DEFAULT_TORCHSTORE_NAME) -> None:
    session = _spmd_state_map.get(store_name)
    if session is not None:
        await session.shutdown()
        return
    controller = await _controller(store_name)
    try:
        await controller.teardown.call()
    finally:
        cl = _local_clent_map.get(store_name)
        if cl is not None:
            state_dict_utils.reset_direct_cache(cl)
            cl.close_sessions()
            cl.strategy.transport_context.clear()
        reset_client(store_name)
        for name in _owned_actors.pop(store_name, []):
            rpc.unregister_actor(name)
        _controllers.pop(store_name, None)


def reset_client(store_name: str = DEFAULT_TORCHSTORE_NAME) -> None:
    _local_clent_map.pop(store_name, None)


async def _controller(store_name: str = DEFAULT_TORCHSTORE_NAME, create: bool = False):
    session = _spmd_state_map.get(store_name)
    if session is not None:
        return session.controller
    ref = _controllers.get(store_name)
    if ref is None:
        if not create:
            raise RuntimeError(f"TorchStore '{store_name}' is not initialized in this process")
        name = f"{store_name}/controller"
        _owned_actors.setdefault(store_name, []).append(name)
        ref = _controllers[store_name] = rpc.register_actor(name, Controller())
    return ref


async def client(store_name: str = DEFAULT_TORCHSTORE_NAME) -> LocalClient:
    cached = _local_clent_map.get(store_name)
    if cached is not None:
        return cached
    controller = await _controller(store_name)
    strategy = await controller.get_controller_strategy.call_one()
    cl = _local_clent_map[store_name] = LocalClient(controller=controller, strategy=strategy)
    return cl


async def put(key: str, value: torch.Tensor | Any, store_name: str = DEFAULT_TORCHSTORE_NAME) -> None:
    return await (await client(store_name)).put(key, value)


async def put_batch(entries: dict[str, torch.Tensor | Any], store_name: str = DEFAULT_TORCHSTORE_NAME, wait: bool = True):
    """``wait=False`` (extension of the reference signature): returns a PendingPut once the copy is
    enqueued on the volume's side stream -- it overlaps the caller's compute; ``await`` it to finish."""
    return await (await client(store_name)).put_batch(entries, wait=wait)


async def get(key: str, inplace_tensor: torch.Tensor | None = None, tensor_slice_spec: TensorSlice | None = None,
              store_name: str = DEFAULT_TORCHSTORE_NAME) -> torch.Tensor | Any:
    return await (await client(store_name)).get(key, inplace_tensor, tensor_slice_spec)


async def get_batch(keys: list[str] | dict[str, torch.Tensor | DTensor | None],
                    store_name: str = DEFAULT_TORCHSTORE_NAME) -> dict[str, Any]:
    return await (await client(store_name)).get_batch(keys)


async def delete(key: str, *, store_name: str = DEFAULT_TORCHSTORE_NAME) -> None:
    return await (await client(store_name=store_name)).delete(key)


async def delete_batch(keys: list[str], *, store_name: str = DEFAULT_TORCHSTORE_NAME) -> None:
    return await (await client(store_name=store_name)).delete_batch(keys)


async def keys(prefix: str | None = None, *, store_name: str = DEFAULT_TORCHSTORE_NAME) -> list[str]:
    return await (await client(store_name=store_name)).keys(prefix)


async def exists(key: str, store_name: str = DEFAULT_TORCHSTORE_NAME) -> bool:
    return await (await client(store_name)).exists(key)


async def put_state_dict(state_dict: dict[str, Any] | None, key: str, store_name: str = DEFAULT_TORCHSTORE_NAME,
                         direct_rdma: bool = False, transfer_dtype: "torch.dtype | None" = None,
                         block_scales: "dict[str, torch.Tensor] | None" = None,
                         channel_scales: "dict[str, torch.Tensor] | None" = None,
                         tensor_scales: "dict[str, torch.Tensor] | None" = None,
                         quantize: "dict[str, str] | None" = None, scale_fmt: "str | None" = None, *,
                         quant_dtype: "torch.dtype | None" = None) -> None:
    cl = await client(store_name)
    await state_dict_utils.put_state_dict(store=cl, state_dict=state_dict, key=key, direct_rdma=direct_rdma,
                                          transfer_dtype=transfer_dtype, block_scales=block_scales,
                                          channel_scales=channel_scales, tensor_scales=tensor_scales,
                                          quantize=quantize, scale_fmt=scale_fmt, quant_dtype=quant_dtype)


async def get_state_dict(key: str, user_state_dict: dict[str, Any] | None = None, strict: bool = True,
                         store_name: str = DEFAULT_TORCHSTORE_NAME, direct_rdma: bool = False,
                         block_scales: "dict[str, torch.Tensor] | None" = None,
                         channel_scales: "dict[str, torch.Tensor] | None" = None,
                         tensor_scales: "dict[str, torch.Tensor] | None" = None,
                         requantize: bool = False, scale_fmt: "str | None" = None,
                         verbatim: bool = False, *, packed: "dict[str, tuple] | None" = None) -> dict[str, Any]:
    cl = await client(store_name)
    return await state_dict_utils.get_state_dict(cl, key, user_state_dict, strict, direct_rdma=direct_rdma,
                                                 block_scales=block_scales, channel_scales=channel_scales,
                                                 tensor_scales=tensor_scales, requantize=requantize,
                                                 scale_fmt=scale_fmt, verbatim=verbatim, packed=packed)

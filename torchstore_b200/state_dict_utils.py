"""State-dict exchange over the store (reference torchstore/state_dict_utils.py:46-212).

Key layout is the reference's: one store key per flattened leaf ``"{key}/{flat_key}"`` and the
mapping object ``"{key}/MAPPING"`` written LAST as the commit marker; direct mode publishes
``"{key}/rank_{r}"`` (that rank's handles) and ``"{key}/num_ranks"``.

``direct_rdma=True`` keeps its name for drop-in compatibility; on this build the "RDMA" is
one-sided P2P reads over NVLink issued by the destination's copy_rects kernel.
"""

from __future__ import annotations

from collections import defaultdict
from dataclasses import dataclass, field
from logging import getLogger
from typing import Any

import torch
import torch.distributed as dist
from torch.distributed.checkpoint._nested_dict import flatten_state_dict, unflatten_state_dict

DELIM = "/"
MAPPING = "MAPPING"

logger = getLogger(__name__)


@dataclass
class _DirectRDMACache:
    """Per-client state of direct weight sync (lazily created halves, published keys, handles)."""

    source: Any = None  # most recently used DirectWeightSyncSource (reference field)
    sources: dict = field(default_factory=dict)  # key -> DirectWeightSyncSource (handles + staging per key)
    dest: Any = None  # most recently used DirectWeightSyncDest (reference field)
    dests: dict = field(default_factory=dict)  # key -> DirectWeightSyncDest (one cached plan per key)
    registered: set = field(default_factory=set)
    handles: dict = field(default_factory=dict)


_rdma_cache: dict[int, _DirectRDMACache] = {}


def _get_rdma_cache(store) -> _DirectRDMACache:
    return _rdma_cache.setdefault(id(store), _DirectRDMACache())


def reset_direct_cache(store=None) -> None:
    """Drop cached plans/handles (called by ``shutdown``; also useful between tests)."""
    keys = list(_rdma_cache) if store is None else [id(store)]
    for k in keys:
        cache = _rdma_cache.pop(k, None)
        if cache is not None:
            for d in cache.dests.values():
                d.close()
            for src in cache.sources.values():
                src._refresh_plans.close()


async def put_state_dict(store, state_dict, key, direct_rdma=False, transfer_dtype=None):
    """Store every leaf of ``state_dict`` (one batched put), then the mapping as the commit marker.

    With ``direct_rdma=True`` only handles to the caller's HBM are published on the first call;
    later calls refresh dtype-cast staging (``state_dict`` may then be None).  ``transfer_dtype``
    applies to direct mode only."""
    if direct_rdma:
        await _put_state_dict_direct_rdma(store, state_dict, key, transfer_dtype)
        return
    flat, mapping = flatten_state_dict(state_dict)
    await store.put_batch({f"{key}{DELIM}{k}": v for k, v in flat.items()})
    await store.put(f"{key}{DELIM}{MAPPING}", mapping)


async def get_state_dict(store, key, user_state_dict: dict | None = None, strict=True, direct_rdma=False):
    """Fetch a state dict.  ``user_state_dict`` tensors are filled in place (and required in direct
    mode).  A missing mapping means no matching push finished: RuntimeError."""
    if direct_rdma:
        assert user_state_dict is not None, "user_state_dict is required for direct_rdma mode"
        await _get_state_dict_direct_rdma(store, key, user_state_dict)
        return user_state_dict
    try:
        fetched_mapping = await store.get(f"{key}{DELIM}{MAPPING}")
    except Exception as e:
        raise RuntimeError(
            f"Mapping is missing from the store. This most likely means there is no matching 'push' call for this key: {key=}"
        ) from e
    user_flat, user_mapping = flatten_state_dict(user_state_dict) if user_state_dict is not None else ({}, None)
    if strict and user_mapping is not None:
        assert user_mapping == fetched_mapping
    wanted = {}
    for flat_key in fetched_mapping.keys():
        target = user_flat.get(flat_key)
        if target is not None and not isinstance(target, torch.Tensor):
            logger.warning("non-tensor value found for in-place: %s", flat_key)
            target = None
        wanted[f"{key}{DELIM}{flat_key}"] = target
    results = await store.get_batch(wanted)
    fetched = {fk: results[f"{key}{DELIM}{fk}"] for fk in fetched_mapping.keys()}
    return unflatten_state_dict(fetched, fetched_mapping)


def _state_dict_size(state_dict) -> int:
    """Size of the tensors of a state dict in MiB."""
    flat, _ = flatten_state_dict(state_dict)
    total = sum(t.numel() * t.element_size() for t in flat.values() if isinstance(t, torch.Tensor))
    return total // (1024 * 1024)


# ---------------------------------------------------------------------------------------------
# direct mode
# ---------------------------------------------------------------------------------------------
async def _put_state_dict_direct_rdma(store, state_dict, key, transfer_dtype=None):
    from torchstore_b200.direct_weight_sync import DirectWeightSyncSource

    cache = _get_rdma_cache(store)
    # one source object per key: the reference keeps a single one per client, whose handles and
    # staging buffers are overwritten when a second key is registered (state_dict_utils.py:171-178)
    cache.source = cache.sources.get(key)
    if cache.source is None:
        cache.source = cache.sources[key] = DirectWeightSyncSource()
    if key not in cache.registered:
        assert state_dict is not None, "state_dict is required on first put_state_dict call with direct_rdma=True"
        rank, world_size = dist.get_rank(), dist.get_world_size()
        handles = cache.source.register(state_dict, rank=rank, transfer_dtype=transfer_dtype)
        await store.put(f"{key}/rank_{rank}", handles)
        if rank == 0:
            await store.put(f"{key}/num_ranks", world_size)
        cache.registered.add(key)
    else:
        cache.source.refresh()
        cache.source.fence()


def _try_all_gather(cache: _DirectRDMACache, key: str, user_state_dict) -> bool:
    """Route "every rank reads every tensor in full from the ranks' own Shard(0) shards" to NCCL's
    all-gather (collectives.py).  All ranks must agree, so the local verdict is min-reduced first."""
    from torch.distributed.tensor import DTensor

    from torchstore_b200.collectives import all_gather_state_dict, is_allgather_shaped

    if not dist.is_initialized() or dist.get_world_size() == 1:
        return False
    rank, world = dist.get_rank(), dist.get_world_size()
    source = cache.sources.get(key)
    ok = source is not None and key in cache.registered and bool(source._handles)
    shards, dests = {}, {}
    if ok:
        ok = not any(isinstance(t, DTensor) for t in user_state_dict.values())
    if ok:
        slices = {n: h.tensor_slice for n, h in source._handles.items()}
        ok = is_allgather_shaped(slices, {n: tuple(t.shape) for n, t in user_state_dict.items()}, rank, world)
    if ok:
        for n, h in source._handles.items():
            shard = h.rdma_buffer._keepalive
            dest = user_state_dict[n]
            if shard is None or shard.dtype != dest.dtype or not dest.is_contiguous():
                ok = False
                break
            shards[n], dests[n] = shard, dest
    device = next(iter(user_state_dict.values())).device if user_state_dict else torch.device("cpu")
    verdict = torch.tensor([1 if ok else 0], device=device if device.type == "cuda" else "cpu")
    dist.all_reduce(verdict, op=dist.ReduceOp.MIN)
    if int(verdict.item()) == 0:
        return False
    all_gather_state_dict(shards, dests)
    return True


async def _get_state_dict_direct_rdma(store, key, user_state_dict):
    from torchstore_b200.collectives import allgather_enabled
    from torchstore_b200.direct_weight_sync import DirectWeightSyncDest

    cache = _get_rdma_cache(store)
    # one destination object (= one cached transfer plan) per state-dict key; the reference keeps a
    # single one per client (state_dict_utils.py:198-201), which silently replays the first key's plan
    # for every later key
    cache.dest = cache.dests.get(key)
    if cache.dest is None:
        cache.dest = cache.dests[key] = DirectWeightSyncDest()
    if allgather_enabled() and _try_all_gather(cache, key, user_state_dict):
        return
    if key not in cache.handles:
        num_ranks = await store.get(f"{key}/num_ranks")
        all_handles = defaultdict(list)
        # one batched fetch of every rank's handle table (the reference does num_ranks sequential gets,
        # state_dict_utils.py:206-209); order by source rank is kept
        tables = await store.get_batch([f"{key}/rank_{r}" for r in range(num_ranks)])
        for r in range(num_ranks):
            for name, handle in tables[f"{key}/rank_{r}"].items():
                all_handles[name].append(handle)
        cache.handles[key] = all_handles
    await cache.dests[key].pull(cache.handles[key], user_state_dict)

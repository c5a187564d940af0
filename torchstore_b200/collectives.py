"""The one place the path uses a collective: "every rank reads the whole key".

When the readers of a sharded state dict are exactly the ranks that hold its FSDP ``Shard(0)``
shards and every reader wants every tensor in full (BASELINE config #3b), the exchange is an
all-gather: rank r contributes rows ``[r*R, (r+1)*R)`` of each tensor and receives the rest.  On an
NVSwitch box NCCL can run that through the switch (NVLS) instead of N-1 point-to-point pulls per
reader, so this case -- and only this case -- is routed to ``torch.distributed``
(``all_gather_into_tensor``; NCCL on GPUs).  Every other layout (resharding, partial readers,
uneven shards) stays on the one-sided copy_rects path.

The reference has no equivalent: each reader fetches all N shards itself
(``client.py:292-314``).  This module is device-agnostic plumbing around the collective, so its
logic is exercised by a world-size-2 gloo test on the CPU; the GPU hot path is NCCL's.

Status: the one-sided pulls need one copy_rects launch per reader where this route needs one NCCL
collective per tensor, so the route stays **off by default** (compare with ``bench.py --config 3b
[--allgather]``; not measured on H100); TORCHSTORE_B200_ALLGATHER=1 selects it.  ``tests/test_gpu_multi.py`` runs it over NCCL on two GPUs.
"""

from __future__ import annotations

import os

import torch
import torch.distributed as dist

from torchstore_b200.transport.types import TensorSlice


def allgather_enabled() -> bool:
    return os.environ.get("TORCHSTORE_B200_ALLGATHER", "0") == "1"


def is_allgather_shaped(local_slices: dict[str, TensorSlice], dest_shapes: dict[str, tuple], rank: int, world: int) -> bool:
    """True when, for every name, the local shard is rows [rank*R, (rank+1)*R) of an evenly
    row-sharded tensor over a 1-D mesh of ``world`` ranks and the destination is the full tensor."""
    if set(local_slices) != set(dest_shapes) or not local_slices:
        return False
    for name, ts in local_slices.items():
        gshape = tuple(ts.global_shape)
        if tuple(dest_shapes[name]) != gshape or len(gshape) == 0:
            return False
        if tuple(ts.mesh_shape) != (world,) or tuple(ts.coordinates) != (rank,):
            return False
        if gshape[0] % world:
            return False
        rows = gshape[0] // world
        if tuple(ts.local_shape) != (rows,) + gshape[1:]:
            return False
        if tuple(ts.offsets) != (rank * rows,) + (0,) * (len(gshape) - 1):
            return False
    return True


def all_gather_state_dict(local_shards: dict[str, torch.Tensor], dests: dict[str, torch.Tensor], group=None) -> int:
    """All-gather every tensor's row shards into its full destination; returns the number of
    collectives issued.  Shards and destinations must be contiguous, same dtype and device kind."""
    pairs = []
    for name, shard in local_shards.items():
        dest = dests[name]
        if not (shard.is_contiguous() and dest.is_contiguous()):
            raise ValueError(f"all_gather_state_dict needs contiguous tensors ({name})")
        if shard.dtype != dest.dtype:
            raise ValueError(f"dtype mismatch for {name}: {shard.dtype} vs {dest.dtype}")
        if dest.numel() != shard.numel() * dist.get_world_size(group):
            raise ValueError(f"shape mismatch for {name}: {tuple(dest.shape)} is not world x {tuple(shard.shape)}")
        pairs.append((dest, shard))
    if not pairs:
        return 0
    if dist.get_backend(group) == "nccl":
        # one NCCL group (ncclGroupStart/End) for the whole state dict instead of a launch per tensor
        try:
            with dist._coalescing_manager(group=group, device=pairs[0][0].device, async_ops=True) as cm:
                for dest, shard in pairs:
                    dist.all_gather_into_tensor(dest, shard, group=group)
            cm.wait()
            return len(pairs)
        except (AttributeError, RuntimeError, TypeError):
            pass  # older torch: fall through to one collective per tensor
    works = [dist.all_gather_into_tensor(dest, shard, group=group, async_op=True) for dest, shard in pairs]
    for w in works:
        w.wait()
    return len(works)

"""Shared setup of the packed-destination tests: FSDP Shard(0) handles over global tensors, the destinations and
``packed`` / ``dest_slices`` arguments of a vLLM TP layout (workloads.vllm_tp_layout), and the unfused pull of
the same bytes into HF-named destinations."""

from __future__ import annotations

import torch

import workloads
from torchstore_b200.direct_weight_sync import RDMAWeightHandle
from torchstore_b200.transport.types import TensorSlice


class HostBuffer:
    """Host-memory stand-in for NvlinkBuffer: the planner reads ``shape`` and ``dtype`` only; ``shard`` is what
    the tests move (None for metadata-only plans)."""

    def __init__(self, shard, shape, dtype):
        self.shard, self.shape, self.dtype = shard, tuple(shape), dtype


def fsdp_handles(layout, n: int, make_buffer, names=None) -> dict[str, list]:
    """Every tensor of ``layout`` cut into ``n`` Shard(0) shards: name -> handles in rank order.
    ``make_buffer(name, offsets, local shape)`` creates each handle's buffer."""
    out = {}
    for name, (shape, _) in layout.items():
        if names is not None and name not in names:
            continue
        hs = []
        for r in range(n):
            off, loc = workloads.shard_box(shape, n, r, ("S", 0)) if n > 1 else ((0,) * len(shape), tuple(shape))
            hs.append(RDMAWeightHandle(make_buffer(name, off, loc), TensorSlice(off, (r,), tuple(shape), loc, (n,)), r))
        out[name] = hs
    return out


def window(full: torch.Tensor, offsets, shape) -> torch.Tensor:
    return full[tuple(slice(o, o + e) for o, e in zip(offsets, shape))]


def pull_args(vlayout, tp: int, rank: int, make_dest):
    """-> (destination dict, dest_slices, packed) of a vLLM layout; ``make_dest(name, local shape)``."""
    dests, slices, packed = {}, {}, {}
    for name, (shape, parts, box) in vlayout.items():
        dests[name] = make_dest(name, shape)
        if parts is None:
            slices[name] = TensorSlice(box[0], (rank,), box[1], tuple(shape), (tp,))
        else:
            packed[name] = parts
    return dests, slices, packed


def unfused_args(vlayout, hf_layout, tp: int, rank: int, make_dest):
    """The same bytes pulled without packing: one HF-named destination per part (its box, at the part's source
    offsets) plus the unpacked names -> (destination dict, dest_slices, {fused name: [(part, unfused name)]})."""
    dests, slices, where = {}, {}, {}
    for name, (shape, parts, box) in vlayout.items():
        if parts is None:
            dests[name] = make_dest(name, shape)
            slices[name] = TensorSlice(box[0], (rank,), box[1], tuple(shape), (tp,))
            continue
        for k, p in enumerate(parts):
            ext = tuple(torch.empty(shape, device="meta")[p.dest_index].shape)
            uname = p.source if p.source not in dests else f"{p.source}#{k}"
            assert uname == p.source, "one unfused destination per source"
            dests[uname] = make_dest(uname, ext)
            slices[uname] = TensorSlice(tuple(p.source_offsets), (rank,), tuple(hf_layout[p.source][0]), ext, (tp,))
            where.setdefault(name, []).append((p, uname))
    return dests, slices, where

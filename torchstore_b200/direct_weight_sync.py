"""Direct weight sync over NVLink -- one hop, one kernel launch per destination GPU.

Same caller-facing surface as the reference's ``torchstore/direct_weight_sync.py``
(RDMAWeightHandle :46-58, DirectWeightSyncSource :82-176, DirectWeightSyncDest :209-350) with
the data plane replaced:

* the ``rdma_buffer`` inside a handle is an :class:`NvlinkBuffer` (exported HBM region + layout;
  picklable; ``read_into`` / ``write_from`` / ``drop`` like ``monarch.rdma.RDMABuffer``);
* the destination does **not** read whole source shards into temporaries and slice afterwards
  (reference :280-286, 3.1x read amplification and 4.8 GB of scratch per rank for Llama-3-8B
  FSDP(8)->TP(8)); every plan op becomes one source-rectangle -> destination-rectangle
  descriptor and the whole plan runs as a single persistent ``copy_rects`` launch that loads
  over NVLink (peer-mapped addresses) and stores coalesced into the destination shard;
* ``transfer_dtype`` staging is refreshed by one batched fused-cast launch instead of one
  ``staging.copy_(src)`` per parameter (reference :158-169); if a handle's dtype differs from the
  destination's, the cast is fused into the gather itself.

Typical usage is unchanged::

    source = DirectWeightSyncSource()
    handles = source.register(model.state_dict(), rank=dist.get_rank())
    await ts.put(f"{RDMA_KEY_PREFIX}/rank_{rank}", handles)
    ...
    dest = DirectWeightSyncDest()
    await dest.pull(all_handles, model.state_dict())
"""

from __future__ import annotations

import logging
from collections import defaultdict
from dataclasses import dataclass

import torch

from torchstore_b200.launch import Plans, copy_once, wait_copy_stream
from torchstore_b200.planner import HbmDescriptor, StridedMem
from torchstore_b200.transport.types import Request, TensorSlice
from torchstore_b200.utils import get_slice_intersection, to_byte_view

logger = logging.getLogger(__name__)

RDMA_KEY_PREFIX = "policy_rdma"


# ---------------------------------------------------------------------------------------------
# the rdma_buffer duck-type
# ---------------------------------------------------------------------------------------------
class NvlinkBuffer:
    """Handle to a contiguous tensor in some GPU's HBM, readable/writable from any GPU on the box.

    Drop-in for the ``rdma_buffer`` field of :class:`RDMAWeightHandle` (reference call sites
    direct_weight_sync.py:143,174,339; monarch_rdma.py:121,146,177).  Pickles to plain bytes.
    """

    def __init__(self, tensor: torch.Tensor | None = None, *, descriptor: HbmDescriptor | None = None):
        if descriptor is None:
            if tensor is None:
                raise ValueError("NvlinkBuffer needs a tensor or a descriptor")
            if not tensor.is_contiguous():
                raise ValueError("NvlinkBuffer registers contiguous memory (stage non-contiguous tensors first)")
            descriptor = HbmDescriptor.from_tensor(tensor)
        self.descriptor = descriptor
        # keep the exporter's tensor alive as long as the handle object lives in its process
        self._keepalive = tensor

    # -- metadata --------------------------------------------------------------------------------
    @property
    def dtype(self) -> torch.dtype:
        return self.descriptor.dtype

    @property
    def shape(self) -> tuple:
        return self.descriptor.shape

    @property
    def nbytes(self) -> int:
        return self.descriptor.nbytes

    @property
    def device(self) -> int:
        return self.descriptor.device

    def __getstate__(self):
        return {"descriptor": self.descriptor}

    def __setstate__(self, state):
        self.descriptor = state["descriptor"]
        self._keepalive = None

    def window(self, device: int) -> StridedMem:
        """The registered tensor as seen from ``device`` (imports + caches the mapping)."""
        return self.descriptor.resolve(device)

    # -- one-sided ops (API parity; the batched plan below is the fast path) ---------------------
    async def read_into(self, dest_byte_view: torch.Tensor) -> None:
        await self._move(dest_byte_view, read=True)

    async def write_from(self, src_byte_view: torch.Tensor) -> None:
        await self._move(src_byte_view, read=False)

    async def _move(self, local_bytes: torch.Tensor, read: bool) -> None:
        if not local_bytes.is_cuda:
            raise RuntimeError("NvlinkBuffer moves bytes between GPUs; got a CPU tensor")
        if local_bytes.dtype != torch.uint8 or local_bytes.dim() != 1 or not local_bytes.is_contiguous():
            raise ValueError("expected a flat contiguous uint8 view (see to_byte_view)")
        if local_bytes.numel() != self.nbytes:
            raise RuntimeError(f"size mismatch: buffer has {self.nbytes} bytes, view has {local_bytes.numel()}")
        device = local_bytes.device.index
        remote = self.window(device).flat_bytes()
        local = StridedMem.from_tensor(local_bytes)
        copy_once({device: [(remote, local) if read else (local, remote)]})
        await wait_copy_stream(device)

    async def drop(self) -> None:
        try:
            self.descriptor.release()
        except Exception as e:  # cleanup failures are logged, not raised (reference monarch_rdma.py:176-179)
            logger.warning("NvlinkBuffer.drop failed: %s", e)
        self._keepalive = None


@dataclass
class RDMAWeightHandle:
    """Serializable handle to one weight shard (same fields as the reference)."""

    rdma_buffer: object  # NvlinkBuffer
    tensor_slice: TensorSlice  # shard position in the global tensor
    source_rank: int


def _request_to_slice(req: Request, param: torch.Tensor) -> TensorSlice:
    """TensorSlice of a request; plain tensors cover their whole (own) global shape at offset 0."""
    if req.tensor_slice is not None:
        return req.tensor_slice
    shape = tuple(param.shape)
    zeros = tuple(0 for _ in shape)
    return TensorSlice(offsets=zeros, coordinates=zeros, global_shape=shape, local_shape=shape,
                       mesh_shape=tuple(1 for _ in shape))


# ---------------------------------------------------------------------------------------------
# source side (trainer)
# ---------------------------------------------------------------------------------------------
class DirectWeightSyncSource:
    """Registers live parameter memory (zero-copy) or dtype-cast staging buffers.

    With ``transfer_dtype`` every param gets an HBM staging buffer in that dtype; ``refresh()``
    re-casts all of them with ONE fused-cast kernel launch per device.
    """

    def __init__(self) -> None:
        self._handles: dict[str, RDMAWeightHandle] = {}
        # name -> (staging_buffer, source_local_tensor)
        self._staging: dict[str, tuple[torch.Tensor, torch.Tensor]] = {}
        self._refresh_plans = Plans()
        self._devices: tuple[int, ...] = ()  # devices holding registered memory (fence targets)

    def register(self, state_dict: dict[str, torch.Tensor], rank: int,
                 transfer_dtype: torch.dtype | None = None,
                 tensor_slices: dict[str, TensorSlice] | None = None) -> dict[str, RDMAWeightHandle]:
        """Create a handle for every entry of ``state_dict`` (tensors or DTensors).

        ``tensor_slices`` (extension) gives the global rectangle of *plain* local shards for
        callers that do not wrap them in DTensors."""
        handles: dict[str, RDMAWeightHandle] = {}
        self._refresh_plans.close()
        self._staging = {}
        casts: dict[int, list] = defaultdict(list)  # device -> (source, staging) windows of the refresh
        devices = set()
        for name, param in state_dict.items():
            req = Request.from_any(name, param, tensor_slices.get(name) if tensor_slices else None)
            local = req.tensor_val
            tslice = _request_to_slice(req, param)
            if not local.is_cuda:
                raise RuntimeError(f"direct weight sync registers GPU memory; '{name}' is on {local.device}")
            devices.add(local.device.index)
            if transfer_dtype is not None:
                staging = torch.empty(local.shape, dtype=transfer_dtype, device=local.device)
                self._staging[name] = (staging, local)
                casts[local.device.index].append((StridedMem.from_tensor(local), StridedMem.from_tensor(staging)))
                buf = staging
            else:
                assert local.is_contiguous(), f"Expected contiguous tensor for key={name}, strides={local.stride()}"
                buf = local
            handles[name] = RDMAWeightHandle(rdma_buffer=NvlinkBuffer(buf), tensor_slice=tslice, source_rank=rank)
        self._handles = handles
        self._devices = tuple(sorted(devices))
        if self._staging:
            self._refresh_plans = Plans.build(casts)
            self.refresh()
        else:
            # make sure the weights the handles point at are materialised before anyone reads them
            for dev in devices:
                torch.cuda.current_stream(dev).synchronize()
        logger.info("Registered %d NVLink handles (%d staged, %d direct)", len(handles), len(self._staging),
                    len(handles) - len(self._staging))
        return handles

    def refresh(self) -> int:
        """Re-cast the source params into their staging buffers (no-op without transfer_dtype).
        Returns the number of staging buffers refreshed.  Blocks until the cast has landed so the
        caller may publish/notify right after, like the reference's synchronous copy loop."""
        if not self._refresh_plans:
            return 0
        self._refresh_plans.launch()
        self._refresh_plans.synchronize()
        return len(self._staging)

    def fence(self) -> None:
        """Make every write queued on the caller's streams (optimizer step, staging refresh) land in
        HBM before readers are told to pull.  The reference has no such fence (its RDMA reads race
        with in-flight kernels); on one box it costs a stream sync."""
        for dev in self._devices:
            torch.cuda.current_stream(dev).synchronize()

    async def cleanup(self) -> None:
        for handle in self._handles.values():
            await handle.rdma_buffer.drop()
        self._handles.clear()
        self._staging.clear()
        self._refresh_plans.close()


# ---------------------------------------------------------------------------------------------
# destination side (generator)
# ---------------------------------------------------------------------------------------------
@dataclass
class _TransferOp:
    """One planned read.  Field names follow the reference (:184-206); ``recv_buffer`` is always
    None here because the kernel reads the overlap rectangle straight from the source shard."""

    rdma_buffer: object
    dest_byte_view: torch.Tensor | None
    dest_tensor: torch.Tensor | None = None  # None <=> exact match (whole shard -> whole param)
    recv_buffer: torch.Tensor | None = None
    src_slices: tuple[slice, ...] | None = None
    dest_slices: tuple[slice, ...] | None = None
    # planner metadata
    name: str = ""
    dest_local: torch.Tensor | None = None


class DirectWeightSyncDest:
    """Pulls weights from source handles with one persistent-kernel launch per local GPU.

    The transfer plan (ops, then the compiled native tile table) is built on the first
    :meth:`pull` and cached, like the reference (:334-335).
    """

    def __init__(self) -> None:
        self._plan: list[_TransferOp] | None = None
        self._plan_signature: tuple | None = None
        self._plan_ids: tuple | None = None  # id() of the destination objects the plan was built for
        self._plan_refs: list | None = None  # ...kept alive, so those ids cannot be recycled
        self._plan_dict: dict | None = None  # the dict object they came in (identity short-cut of the next pull)
        self._native_plans = Plans()  # the compiled plan, one native plan per destination device
        self.last_pull_ms: dict[int, float] = {}  # device -> kernel time of the last pull

    # -- planning (host, metadata only) ----------------------------------------------------------
    def _build_plan(self, all_handles: dict[str, list[RDMAWeightHandle]],
                    dest_state_dict: dict[str, torch.Tensor],
                    dest_slices: dict[str, TensorSlice] | None = None) -> list[_TransferOp]:
        """Per destination param x per source handle: intersect, dedup replicated regions, classify
        exact / partial (same rules and op order as the reference, :221-317).

        ``dest_slices`` (extension) names the rectangle a *plain* local tensor holds, for callers
        that keep raw shards instead of DTensors (e.g. torchrun ranks)."""
        ops: list[_TransferOp] = []
        for name, param in dest_state_dict.items():
            handles = all_handles.get(name)
            if not handles:
                continue
            override = dest_slices.get(name) if dest_slices else None
            dest_req = Request.from_any(name, param, override)
            dest_tensor = dest_req.tensor_val
            dest_slice = _request_to_slice(dest_req, param)
            seen: set[tuple] = set()  # replicated sources: read each region once
            for handle in handles:
                inter = get_slice_intersection(handle.tensor_slice, dest_slice)
                if inter is None:
                    continue
                region = (inter.offsets, inter.local_shape)
                if region in seen:
                    continue
                seen.add(region)
                src_slice = handle.tensor_slice
                exact = src_slice.offsets == dest_slice.offsets and src_slice.local_shape == dest_slice.local_shape
                if exact:
                    assert dest_tensor.is_contiguous(), (
                        f"Expected contiguous dest tensor for key={name}, strides={dest_tensor.stride()}"
                    )
                    ops.append(_TransferOp(rdma_buffer=handle.rdma_buffer, dest_byte_view=to_byte_view(dest_tensor),
                                           name=name, dest_local=dest_tensor))
                else:
                    ndim = len(inter.offsets)
                    src_idx = tuple(
                        slice(inter.offsets[d] - src_slice.offsets[d],
                              inter.offsets[d] - src_slice.offsets[d] + inter.local_shape[d])
                        for d in range(ndim)
                    )
                    dst_idx = tuple(
                        slice(inter.offsets[d] - dest_slice.offsets[d],
                              inter.offsets[d] - dest_slice.offsets[d] + inter.local_shape[d])
                        for d in range(ndim)
                    )
                    ops.append(_TransferOp(rdma_buffer=handle.rdma_buffer, dest_byte_view=None, dest_tensor=dest_tensor,
                                           src_slices=src_idx, dest_slices=dst_idx, name=name, dest_local=dest_tensor))
        logger.info("Built transfer plan with %d NVLink ops", len(ops))
        return ops

    @staticmethod
    def op_windows(op: _TransferOp, src_window: StridedMem) -> tuple[StridedMem, StridedMem]:
        """(source rectangle, destination rectangle) of one op given the mapped source shard."""
        dst_full = StridedMem.from_tensor(op.dest_local)
        if op.dest_tensor is None:
            # exact: whole shard onto whole param (reshape of the source is irrelevant: same numel)
            src = src_window
            if tuple(src.shape) != tuple(dst_full.shape):
                src = StridedMem(src.ptr, dst_full.shape, _contig(dst_full.shape), src.dtype, src.device)
            return src, dst_full
        return src_window.sub(op.src_slices), dst_full.sub(op.dest_slices)

    @staticmethod
    def _signature(dest_state_dict) -> tuple:
        # data pointers only: ~35 us for 291 tensors; a new state_dict() wrapper around the same
        # memory keeps the plan, new memory invalidates it
        return tuple(getattr(p, "_local_tensor", p).data_ptr() for p in dest_state_dict.values())

    def _compile(self) -> None:
        per_device: dict[int, list] = defaultdict(list)
        for op in self._plan:
            dest = op.dest_local
            if not dest.is_cuda:
                raise RuntimeError(
                    f"direct weight sync writes GPU memory; destination '{op.name}' is on {dest.device} "
                    "(torchstore_b200 has no CPU data path)"
                )
            if not isinstance(op.rdma_buffer, NvlinkBuffer):
                raise TypeError(
                    f"handle for '{op.name}' carries a {type(op.rdma_buffer).__name__}; the direct path needs NvlinkBuffer handles"
                )
            dev = dest.device.index
            per_device[dev].append(self.op_windows(op, op.rdma_buffer.window(dev)))
        self._native_plans = Plans.build(per_device)

    def plan_info(self) -> dict[int, dict]:
        return self._native_plans.info()

    # -- execution ---------------------------------------------------------------------------------
    async def pull(self, all_handles: dict[str, list[RDMAWeightHandle]],
                   dest_state_dict: dict[str, torch.Tensor],
                   dest_slices: dict[str, TensorSlice] | None = None) -> None:
        """Pull every overlapping region into ``dest_state_dict`` (in place).  Returns when the
        bytes are in destination HBM (so the caller may tell the source it is done reading).

        Steady state costs one native call to launch and a poll loop: the cached plan is checked
        against the destination OBJECTS first (their ids; the plan keeps them alive), the kernel
        is enqueued, and the data-pointer signature -- which catches ``param.data = new`` under an
        unchanged object -- is recomputed while the kernel runs."""
        if self._plan is not None and dest_state_dict is self._plan_dict:
            # the very dict object of the last pull: launch first, validate it (object ids, then data pointers)
            # while the kernel runs -- a stale launch only fills memory the plan still references
            self.launch()
            same = tuple(map(id, dest_state_dict.values())) == self._plan_ids and \
                self._signature(dest_state_dict) == self._plan_signature
            await self.wait()
            if same:
                return
            logger.info("destination dict was edited in place; rebuilding the transfer plan")
            self.close()
        ids = tuple(map(id, dest_state_dict.values()))
        verified = False
        if self._plan is not None and ids != self._plan_ids:
            # other wrapper objects: fine if they alias the same memory (e.g. a fresh state_dict())
            if self._signature(dest_state_dict) != self._plan_signature:
                logger.info("destination tensors changed; rebuilding the transfer plan")
                self.close()
            else:
                self._plan_ids, self._plan_refs, self._plan_dict = ids, list(dest_state_dict.values()), dest_state_dict
            verified = True
        if self._plan is None:
            self._plan = self._build_plan(all_handles, dest_state_dict, dest_slices)
            self._compile()
            self._plan_signature = self._signature(dest_state_dict)
            self._plan_ids, self._plan_refs, self._plan_dict = ids, list(dest_state_dict.values()), dest_state_dict
            verified = True
        self.launch()
        stale = not verified and self._signature(dest_state_dict) != self._plan_signature
        await self.wait()
        if stale:
            # the launch above filled the OLD memory (still referenced by the plan, so harmless)
            logger.info("destination storage changed under the same tensors; rebuilding the transfer plan")
            self.close()
            await self.pull(all_handles, dest_state_dict, dest_slices)

    def launch(self) -> None:
        """Enqueue the cached plan on each device's copy stream, fenced against the caller's current
        stream on both sides (later work on that stream sees the new weights without a host wait)."""
        if self._plan is None:
            raise RuntimeError("pull() must build the plan first")
        self._native_plans.launch()

    async def wait(self) -> None:
        await self._native_plans.wait()
        self.last_pull_ms.update(self._native_plans.elapsed_ms())

    def close(self) -> None:
        self._native_plans.close()
        self._plan = None
        self._plan_ids = self._plan_refs = self._plan_dict = None


def _contig(shape) -> tuple:
    out, s = [], 1
    for e in reversed(shape):
        out.append(s)
        s *= e
    return tuple(reversed(out))

"""NVLink / HBM transport: the storage-volume data plane of this build.

Implements the ``TransportBuffer`` contract (transport/buffers.py) the way the reference's
``SharedMemoryTransportBuffer`` does (transport/shared_memory.py:263-483), with HBM instead of
POSIX shm and the copy_rects kernel instead of ``Tensor.copy_``.  The landing-buffer put protocol
is ``LandingBufferTransport``'s; this module supplies the HBM memory and the copies:

PUT  1. volume   recv_handshake: the stored CUDA tensor when shape, dtype and contiguity match
                 (overwrite in place), else a new one from the volume's HBM arena; objects -> None
     2. client   _post_handshake: ONE copy_rects launch pushes every tensor of the batch into the
                 volume's memory (local D2D when the volume is on the caller's GPU, P2P stores over
                 NVLink otherwise; host tensors go through an async H2D copy); awaits completion
     3. volume   handle_put_request: stores the landing buffers / objects
GET  1. volume   handle_get_request: descriptor (exported region + layout) of each stored CUDA view
     2. client   _handle_storage_volume_response: ONE copy_rects launch gathers every requested
                 rectangle straight into the caller's tensors (strided destinations included;
                 a dtype pair the fused cast lacks lands in a temporary and is converted by copy_);
                 without a destination the result is materialised on the host like the reference
                 does (D2H), or on the GPU when TORCHSTORE_B200_GET_DEVICE=cuda
"""

from __future__ import annotations

import logging
import os
import weakref
from typing import TYPE_CHECKING, Any

import torch

from torchstore_b200 import _native
from torchstore_b200.launch import Plans, copy_once, staging_copy, wait_copy_stream
from torchstore_b200.logging import LatencyTracker
from torchstore_b200.planner import HbmDescriptor, StridedMem
from torchstore_b200.transport.buffers import EntryContext, LandingBufferTransport, TransportBuffer, TransportCache
from torchstore_b200.transport.types import Request

if TYPE_CHECKING:
    from torchstore_b200.strategy import StorageVolumeRef
    from torchstore_b200.transport.buffers import TransportContext

logger = logging.getLogger(__name__)


def get_result_device() -> str:
    return os.environ.get("TORCHSTORE_B200_GET_DEVICE", "cpu")


# ---------------------------------------------------------------------------------------------
# volume-side memory: HBM arenas
# ---------------------------------------------------------------------------------------------
class _ArenaBlock:
    """Owner of one arena allocation; exposes it to torch through __cuda_array_interface__ and
    returns it to the arena when the last tensor view dies."""

    def __init__(self, arena: int, ptr: int, nbytes: int):
        self.ptr = ptr
        self.nbytes = nbytes
        self.__cuda_array_interface__ = {
            "shape": (max(nbytes, 1),),
            "typestr": "|u1",
            "data": (ptr, False),
            "version": 2,
            "strides": None,
        }
        weakref.finalize(self, _free_block, arena, ptr)


def _free_block(arena: int, ptr: int) -> None:
    try:
        _native.arena_free(arena, ptr)
    except Exception:  # arena already destroyed at shutdown
        pass


class HbmPool:
    """Grow-on-demand list of arena slabs (one cudaMalloc each) on one device."""

    def __init__(self, device: int, slab_bytes: int | None = None):
        self.device = device
        self.slab_bytes = slab_bytes or int(os.environ.get("TORCHSTORE_B200_SLAB_BYTES", 4 << 30))
        self.arenas: list[int] = []

    def alloc_tensor(self, shape, dtype: torch.dtype) -> torch.Tensor:
        numel = 1
        for s in shape:
            numel *= s
        nbytes = numel * dtype.itemsize
        ptr = arena = None
        for a in reversed(self.arenas):
            try:
                ptr, arena = _native.arena_alloc(a, max(nbytes, 1)), a
                break
            except _native.TsbError as e:
                if e.code != _native.TSB_ERR_NOMEM:
                    raise
        if ptr is None:
            mib = 1 << 20
            arena = _native.arena_create(self.device, max(self.slab_bytes, (nbytes + mib) // mib * mib))
            self.arenas.append(arena)
            ptr = _native.arena_alloc(arena, max(nbytes, 1))
        block = _ArenaBlock(arena, ptr, nbytes)
        flat = torch.as_tensor(block, device=torch.device("cuda", self.device))
        return flat[:nbytes].view(dtype).reshape(tuple(shape))

    def stats(self) -> dict:
        out = {"slabs": len(self.arenas), "capacity": 0, "in_use": 0, "high_water": 0}
        for a in self.arenas:
            st = _native.arena_stats(a)
            out["capacity"] += st.capacity
            out["in_use"] += st.in_use
            out["high_water"] += st.high_water
        return out

    def close(self) -> None:
        import gc

        gc.collect()
        for a in self.arenas:
            try:
                _native.arena_destroy(a)
            except Exception as e:
                logger.warning("arena_destroy failed: %s", e)
        self.arenas = []


class HbmVolumeCache(TransportCache):
    """Volume-side long-lived state: the HBM pool stored tensors are carved from."""

    def __init__(self) -> None:
        self.device: int | None = None
        self._pool: HbmPool | None = None

    def configure(self, device: int | None) -> None:
        self.device = device

    def allocate(self, shape, dtype: torch.dtype) -> torch.Tensor:
        if self.device is None:
            raise RuntimeError(
                "this storage volume has no GPU: torchstore_b200 keeps tensors in HBM and has no host-memory "
                "fallback (objects can still be stored)"
            )
        if self._pool is None:
            self._pool = HbmPool(self.device)
        return self._pool.alloc_tensor(shape, dtype)

    def stats(self) -> dict:
        return self._pool.stats() if self._pool is not None else {"slabs": 0, "capacity": 0, "in_use": 0, "high_water": 0}

    def clear(self) -> None:
        if self._pool is not None:
            self._pool.close()
            self._pool = None


class HbmClientCache(TransportCache):
    """Client-side long-lived state.  Region mappings are cached natively per
    (exporter, allocation); clearing the context drops them all
    (reference SharedMemoryCache.clear, shared_memory.py:246-250)."""

    def clear(self) -> None:
        try:
            _native.release_all()
        except Exception as e:
            logger.warning("release_all failed: %s", e)


class HbmTransportBuffer(LandingBufferTransport):
    # the reshard kernel writes strided destination rectangles directly, so the client may hand
    # non-contiguous in-place views (the reference restricts to contiguous ones, utils.py:94-96)
    supports_strided_inplace = True
    supports_fast_lane = True

    def __init__(self, storage_volume_ref: "StorageVolumeRef"):
        super().__init__(storage_volume_ref)
        self.record = False           # client: compile Plans for the fast lane instead of one-shot copies
        self._recorded_plans: Plans | None = None

    # ---- volume memory: HBM arenas --------------------------------------------------------------
    def _describe(self, ctx: "TransportContext", tensor: torch.Tensor) -> HbmDescriptor | None:
        return HbmDescriptor.from_tensor(tensor) if tensor.is_cuda else None

    def _allocate(self, ctx: "TransportContext", shape: tuple, dtype: torch.dtype) -> tuple[torch.Tensor, HbmDescriptor]:
        tensor = ctx.get(HbmVolumeCache).allocate(shape, dtype)
        return tensor, HbmDescriptor.from_tensor(tensor)

    # ---- PUT ------------------------------------------------------------------------------------
    async def _post_handshake(self, handshake_results: list[Any], requests: list[Request]) -> None:
        """Client: move the batch into the volume's HBM with one launch (+ H2D for host tensors)."""
        tracker = LatencyTracker("post_handshake")
        self.storage_volume_ref.transport_context.get(HbmClientCache)
        self._contexts = []
        per_device: dict[int, list] = {}
        host_copies = []
        keep = []
        for request, desc in zip(requests, handshake_results, strict=True):
            if request.is_object:
                self._contexts.append(EntryContext(objects=request.objects, use_rpc=True))
                continue
            tensor = request.tensor_val
            assert tensor is not None and desc is not None
            self._contexts.append(EntryContext(descriptor=desc))
            if tensor.is_cuda:
                dev = tensor.device.index
                per_device.setdefault(dev, []).append((StridedMem.from_tensor(tensor), desc.resolve(dev)))
            else:
                src = tensor if tensor.is_contiguous() else tensor.contiguous()
                keep.append(src)
                host_copies.append((src, desc))
        tracker.track_step("plan")
        devices = self._copy(per_device, record=self.record and not host_copies, fence_out=False)
        for src, desc in host_copies:
            dev = desc.device if _same_process(desc) else torch.cuda.current_device()
            dst = desc.resolve(dev)
            staging_copy(dev, dst.ptr, src.data_ptr(), src.numel() * src.element_size(), _native.TSB_H2D)
            devices.add(dev)
        tracker.track_step("alloc_and_copy")
        for dev in devices:
            await wait_copy_stream(dev)
        tracker.track_step("cuda_synchronize")

    def _copy(self, per_device: dict[int, list], record: bool, fence_out: bool) -> set[int]:
        """One launch per device; a recorded batch keeps its compiled plans for the next identical
        batch to replay.  Returns the devices to wait on."""
        if not (record and per_device):
            return copy_once(per_device)
        self._recorded_plans = Plans.build(per_device)
        self._recorded_plans.launch(fence_out)
        return set(per_device)

    # ---- GET ------------------------------------------------------------------------------------
    async def _handle_storage_volume_response(self, requests: list[Request], transport_buffer: "TransportBuffer") -> list[Any]:
        self.storage_volume_ref.transport_context.get(HbmClientCache)
        results: list[Any] = [None] * len(requests)
        per_device: dict[int, list] = {}
        d2h = []
        converts = []  # (CUDA destination, gathered stored-dtype temporary) for pairs the fused cast lacks
        for i, (request, hctx) in enumerate(zip(requests, transport_buffer._contexts, strict=True)):
            dest = request.tensor_val
            if hctx.use_rpc:
                data = hctx.objects
                if isinstance(data, torch.Tensor) and dest is not None:
                    raise RuntimeError("unexpected host tensor in an HBM volume response")
                results[i] = data
                continue
            desc = hctx.descriptor
            assert desc is not None, f"No descriptor or data for key {request.key}"
            gather = getattr(request, "_gather", None)
            if dest is None and gather is not None:
                # part of a sharded key fetched without a destination: land in the shared GPU
                # bounding-box buffer (replaces the reference's CPU assemble_tensor, utils.py:158-212)
                dest = gather.view_for(request.tensor_slice, desc.dtype, torch.device("cuda", torch.cuda.current_device()))
            if dest is not None:
                assert tuple(dest.shape) == tuple(desc.shape), f"{tuple(dest.shape)} != {tuple(desc.shape)}"
                if dest.is_cuda:
                    dev = dest.device.index
                    target = dest
                    if not _native.cast_supported(desc.dtype, dest.dtype):
                        # no fused cast for this pair: gather the stored dtype in the same launch, then
                        # convert like the reference's client_tensor.copy_(shm_tensor)
                        target = torch.empty(desc.shape, dtype=desc.dtype, device=dest.device)
                        converts.append((dest, target))
                    per_device.setdefault(dev, []).append((desc.resolve(dev), StridedMem.from_tensor(target)))
                    results[i] = dest
                else:
                    d2h.append((i, desc, dest))
            elif get_result_device() == "cuda":
                dev = torch.cuda.current_device()
                out = torch.empty(desc.shape, dtype=desc.dtype, device=torch.device("cuda", dev))
                per_device.setdefault(dev, []).append((desc.resolve(dev), StridedMem.from_tensor(out)))
                results[i] = out
            else:
                d2h.append((i, desc, None))
        self._volume_epoch = transport_buffer._volume_epoch
        # a batch with host results, or one finished by a torch conversion after the plan, is not replayable
        devices = self._copy(per_device, record=self.record and not d2h and not converts, fence_out=True)
        staged = []
        for i, desc, dest in d2h:
            dev = desc.device if _same_process(desc) else torch.cuda.current_device()
            src = desc.resolve(dev)
            # host destination: gather into a contiguous HBM bounce when the stored view is strided,
            # then one D2H copy
            if not src.is_contiguous():
                bounce = torch.empty(desc.shape, dtype=desc.dtype, device=torch.device("cuda", dev))
                copy_once({dev: [(src, StridedMem.from_tensor(bounce))]}, fence=False)
                src_ptr = bounce.data_ptr()
            else:
                bounce, src_ptr = None, src.ptr
            # raw stored bytes may only land in a host tensor of the SAME dtype and size; anything else
            # goes through a temporary and a converting copy_ (what the reference's
            # client_tensor.copy_(shm_tensor) does, shared_memory.py:473-476) -- never a memcpy of
            # desc.nbytes into a buffer of another size
            direct = dest is not None and dest.is_contiguous() and dest.dtype == desc.dtype and \
                dest.numel() * dest.element_size() == desc.nbytes
            host = dest if direct else torch.empty(desc.shape, dtype=desc.dtype)
            staging_copy(dev, host.data_ptr(), src_ptr, desc.nbytes, _native.TSB_D2H)
            devices.add(dev)
            staged.append((i, dest, host, bounce))
        for dev in devices:
            await wait_copy_stream(dev)
        for dest, gathered in converts:
            dest.copy_(gathered)
        for i, dest, host, _bounce in staged:
            if dest is not None and host is not dest:
                dest.copy_(host)  # non-contiguous host destination: host-side scatter of host data
                results[i] = dest
            else:
                results[i] = host
        return results

    def take_recorded(self) -> tuple[Plans, int] | None:
        """Client, after a recorded put or get: the compiled plans and the volume epoch they were built
        under, or None with the plans closed when the request never got an epoch (it failed)."""
        plans, self._recorded_plans = self._recorded_plans, None
        if plans is not None and self._volume_epoch is None:
            plans.close()
            plans = None
        return None if plans is None else (plans, int(self._volume_epoch))


def _same_process(desc: HbmDescriptor) -> bool:
    region = _native.region_from_bytes(desc.region)
    return region.pid == os.getpid()

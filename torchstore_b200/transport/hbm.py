"""NVLink / HBM transport: the storage-volume data plane of this build.

Implements the ``TransportBuffer`` contract (transport/buffers.py) the way the reference's
``SharedMemoryTransportBuffer`` does (transport/shared_memory.py:263-483), with HBM instead of
POSIX shm and the copy_rects kernel instead of ``Tensor.copy_``:

PUT  1. client   requires_handshake: any tensor in the batch -> yes; records (shape, dtype) per entry
     2. volume   recv_handshake: descriptor of the existing stored tensor when shape/dtype match
                 (overwrite in place), else allocate from the volume's HBM arena; objects -> None
     3. client   _post_handshake: ONE copy_rects launch pushes every tensor of the batch into the
                 volume's memory (local D2D when the volume is on the caller's GPU, P2P stores over
                 NVLink otherwise; host tensors go through an async H2D copy); awaits completion
     4. volume   handle_put_request: returns the stored tensors / objects, aligned with entries
GET  1. volume   handle_get_request: descriptor (exported region + layout) of each stored view
     2. client   _handle_storage_volume_response: ONE copy_rects launch gathers every requested
                 rectangle straight into the caller's tensors (strided destinations included);
                 without a destination the result is materialised on the host like the reference
                 does (D2H), or on the GPU when TORCHSTORE_B200_GET_DEVICE=cuda
"""

from __future__ import annotations

import logging
import os
import time
import weakref
from dataclasses import dataclass
from typing import TYPE_CHECKING, Any

import torch

from torchstore_b200 import _native
from torchstore_b200.launch import Plans, copy_once, wait_copy_stream
from torchstore_b200.logging import LatencyTracker
from torchstore_b200.planner import HbmDescriptor, StridedMem
from torchstore_b200.transport.buffers import TransportBuffer, TransportCache
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

    def configure(self, device: int | None, store=None) -> None:
        self.device = device
        self._store = store

    def epoch_of_store(self) -> int | None:
        store = getattr(self, "_store", None)
        return None if store is None else store.epoch

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


# ---------------------------------------------------------------------------------------------
# per-entry state carried inside the pickled buffer
# ---------------------------------------------------------------------------------------------
@dataclass
class HbmContext:
    descriptor: HbmDescriptor | None = None
    objects: Any = None
    use_rpc: bool = False  # objects (and anything that is not an HBM tensor) ride in the RPC


@dataclass
class _PutSpec:
    shape: tuple
    dtype: torch.dtype


class HbmTransportBuffer(TransportBuffer):
    supports_inplace_resharding = True
    supports_batch_puts = True
    supports_batch_gets = True
    # the reshard kernel writes strided destination rectangles directly, so the client may hand
    # non-contiguous in-place views (the reference restricts to contiguous ones, utils.py:94-96)
    supports_strided_inplace = True
    supports_fast_lane = True

    def __init__(self, storage_volume_ref: "StorageVolumeRef"):
        super().__init__(storage_volume_ref)
        self._needs_handshake = False
        self._contexts: list[HbmContext] = []
        self._put_specs: list[_PutSpec | None] = []
        # identifies THIS put on the volume between handshake and put (two clients may put the same
        # key concurrently; each must get back the landing buffer it wrote into)
        self._nonce = os.urandom(8).hex()
        self._epoch = None            # volume layout epoch seen by the volume half of a get, or after a put
        self.record = False           # client: compile Plans for the fast lane instead of one-shot copies
        self._recorded_plans: Plans | None = None

    def __getstate__(self) -> dict[str, Any]:
        state = self.__dict__.copy()
        state["storage_volume_ref"] = None  # process-local handle
        return state

    # ---- PUT ------------------------------------------------------------------------------------
    def requires_handshake(self, requests: list[Request]) -> bool:
        if not self._needs_handshake:
            return False
        self._put_specs = [
            None if r.is_object else _PutSpec(tuple(r.tensor_val.shape), r.tensor_val.dtype) for r in requests
        ]
        return True

    async def put_to_storage_volume(self, requests: list[Request]) -> None:
        self._needs_handshake = True
        await super().put_to_storage_volume(requests)
        self._epoch = self._volume_epoch

    async def recv_handshake(self, ctx: "TransportContext", entries: list[tuple[Request, Any]]) -> list[Any]:
        """Volume: hand out where each tensor must be written."""
        vol = ctx.get(HbmVolumeCache)
        out: list[HbmDescriptor | None] = []
        pending = _pending(ctx)
        _purge_stale(pending)
        for idx, ((request, current), spec) in enumerate(zip(entries, self._put_specs, strict=True)):
            if spec is None:
                out.append(None)
                continue
            if isinstance(current, torch.Tensor) and tuple(current.shape) == spec.shape and current.dtype == spec.dtype \
                    and current.is_contiguous():
                target = current  # overwrite in place (reference storage_volume.py:161-207)
            else:
                target = vol.allocate(spec.shape, spec.dtype)
            # keep new allocations alive until handle_put_request stores them
            pending[(self._nonce, idx)] = (time.monotonic(), target)
            out.append(HbmDescriptor.from_tensor(target))
        return out

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
                self._contexts.append(HbmContext(objects=request.objects, use_rpc=True))
                continue
            tensor = request.tensor_val
            assert tensor is not None and desc is not None
            self._contexts.append(HbmContext(descriptor=desc))
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
            _native.memcpy_async(dev, dst.ptr, src.data_ptr(), src.numel() * src.element_size(), _native.TSB_H2D)
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

    async def handle_put_request(self, ctx: "TransportContext", entries: list[tuple[Request, Any]]) -> list[Any]:
        results = []
        pending = _pending(ctx)
        for idx, ((request, current), hctx) in enumerate(zip(entries, self._contexts, strict=True)):
            if hctx.use_rpc:
                results.append(hctx.objects)
                continue
            entry = pending.pop((self._nonce, idx), None)
            assert entry is not None, f"No landing buffer for {request.key}: put without a matching handshake"
            results.append(entry[1])
        return results

    # ---- GET ------------------------------------------------------------------------------------
    async def handle_get_request(self, ctx: "TransportContext", entries: list[tuple[Request, Any]]) -> None:
        self._contexts = []
        self._epoch = ctx.get(HbmVolumeCache).epoch_of_store()
        for request, data in entries:
            if request.is_object or not isinstance(data, torch.Tensor):
                self._contexts.append(HbmContext(objects=data, use_rpc=True))
            elif data.is_cuda:
                self._contexts.append(HbmContext(descriptor=HbmDescriptor.from_tensor(data)))
            else:
                self._contexts.append(HbmContext(objects=data, use_rpc=True))

    async def _handle_storage_volume_response(self, requests: list[Request], transport_buffer: "TransportBuffer") -> list[Any]:
        self.storage_volume_ref.transport_context.get(HbmClientCache)
        results: list[Any] = [None] * len(requests)
        per_device: dict[int, list] = {}
        d2h = []
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
                    per_device.setdefault(dev, []).append((desc.resolve(dev), StridedMem.from_tensor(dest)))
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
        self._epoch = transport_buffer._epoch
        # a batch with host results is not replayable
        devices = self._copy(per_device, record=self.record and not d2h, fence_out=True)
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
            _native.memcpy_async(dev, host.data_ptr(), src_ptr, desc.nbytes, _native.TSB_D2H)
            devices.add(dev)
            staged.append((i, dest, host, bounce))
        for dev in devices:
            await wait_copy_stream(dev)
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
        if plans is not None and self._epoch is None:
            plans.close()
            plans = None
        return None if plans is None else (plans, int(self._epoch))

    async def drop(self) -> None:
        self._contexts = []
        self._put_specs = []


# volume-side scratch: landing buffers between handshake and put, kept on the volume cache object
def _pending(ctx: "TransportContext") -> dict:
    vol = ctx.get(HbmVolumeCache)
    if not hasattr(vol, "_pending"):
        vol._pending = {}
    return vol._pending


_PENDING_TTL_S = 300.0


def _purge_stale(pending: dict) -> None:
    """Landing buffers of puts that failed between handshake and put (the client's drop() cannot
    reach the volume) go back to the arena after a grace period."""
    if not pending:
        return
    now = time.monotonic()
    for k in [k for k, (t, _) in pending.items() if now - t > _PENDING_TTL_S]:
        pending.pop(k, None)


def _same_process(desc: HbmDescriptor) -> bool:
    region = _native.region_from_bytes(desc.region)
    return region.pid == os.getpid()

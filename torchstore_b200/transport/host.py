"""Host tier (SURVEY.md section 8, row f4): POSIX shared-memory volumes for CPU clients and GPU-less
boxes -- the reference's ``SharedMemoryTransportBuffer`` (transport/shared_memory.py:263-483)
rebuilt on the C-ABI's ``tsb_shm_*`` / ``tsb_host_copy_rects`` entry points.

Selected by ``TransportType.SharedMemory`` (the reference's own member name), or automatically when
the client process has no CUDA device at all (BASELINE config #1: "CPU/POSIX-shm, plumbing, no GPU").
It is a tier, not a fallback: on a GPU box the default stays the NVLink/HBM transport, GPU tensors
put through THIS transport are staged with explicit D2H/H2D copies like the reference does
(:374,:475), and nothing in the HBM path ever routes here.

PUT  handshake (``LandingBufferTransport``, shared with the HBM transport): the volume allocates one
     shm segment per tensor (or reuses the stored one when shape, dtype and contiguity match:
     in-place overwrite, storage_volume.py:161-207) and returns its descriptor; the client
     attaches (cached) and moves the bytes in with ONE threaded ``tsb_host_copy_rects`` call for
     all CPU tensors of the batch (strided sources included) and async D2H copies for CUDA tensors.
GET  the volume returns descriptors of the stored views; the client copies segment -> destination
     (strided CPU destinations in place, CUDA destinations by H2D), or hands back a private clone
     when no destination was given (the reference's TORCHSTORE_MUTABLE_SHM=0 behaviour, :478).
"""

from __future__ import annotations

import bisect
import ctypes
import logging
import os
import threading
import weakref
from dataclasses import dataclass
from typing import TYPE_CHECKING, Any

import torch

from torchstore_b200 import _native
from torchstore_b200.launch import staging_copy, wait_copy_stream
from torchstore_b200.planner import StridedMem, build_rects
from torchstore_b200.transport.buffers import EntryContext, LandingBufferTransport, TransportBuffer, TransportCache
from torchstore_b200.transport.types import Request

if TYPE_CHECKING:
    from torchstore_b200.transport.buffers import TransportContext

logger = logging.getLogger(__name__)

_COPY_THREADS = int(os.environ.get("TORCHSTORE_B200_HOST_THREADS", str(min(16, os.cpu_count() or 1))))
_seq = [0]
_seq_lock = threading.Lock()


def _wrap(ptr: int, nbytes: int, shape, stride, dtype: torch.dtype, storage_offset: int = 0) -> torch.Tensor:
    """torch view of mapped memory (no copy); the mapping is owned by the cache that made it."""
    raw = (ctypes.c_char * max(nbytes, 1)).from_address(ptr)
    flat = torch.frombuffer(raw, dtype=torch.uint8, count=max(nbytes, 1))[:nbytes]
    base = flat.view(dtype) if nbytes else torch.empty(0, dtype=dtype)
    return torch.as_strided(base, tuple(shape), tuple(stride), storage_offset)


@dataclass(frozen=True)
class ShmDescriptor:
    """Where a stored tensor (or a view of one) lives: segment + layout.  Picklable."""

    name: str
    segment_bytes: int
    shape: tuple
    stride: tuple  # elements
    dtype: torch.dtype
    storage_offset: int = 0  # elements from the start of the segment

    @property
    def nbytes(self) -> int:
        n = self.dtype.itemsize
        for s in self.shape:
            n *= s
        return n


class _Segment:
    def __init__(self, name: str, ptr: int, nbytes: int, owner: bool):
        self.name, self.ptr, self.nbytes, self.owner = name, ptr, nbytes, owner
        self.registered = False

    def pin(self) -> None:
        """Page-lock for async H2D/D2H when a GPU is around (reference pin_memory, :55-96)."""
        if not self.registered and torch.cuda.is_available():
            try:
                _native.host_register(self.ptr, self.nbytes)
                self.registered = True
            except Exception as e:  # pinning is an optimisation
                logger.debug("host_register failed: %s", e)

    def close(self) -> None:
        if self.registered:
            try:
                _native.host_unregister(self.ptr)
            except Exception:
                pass
            self.registered = False
        try:
            _native.shm_detach(self.ptr, self.nbytes)
        except Exception as e:
            logger.warning("shm_detach(%s) failed: %s", self.name, e)
        if self.owner:
            try:
                _native.shm_unlink(self.name)
            except Exception as e:
                logger.warning("shm_unlink(%s) failed: %s", self.name, e)


class HostVolumeCache(TransportCache):
    """Volume side: the segments this volume owns (created at handshake, unlinked on clear)."""

    def __init__(self) -> None:
        self.segments: dict[str, _Segment] = {}
        self._storage_refs: dict[str, weakref.ref] = {}  # segment name -> weakref on the stored tensor's storage
        self._starts: list[int] = []                     # sorted base addresses of our segments (describe() bisects)
        self._by_start: dict[int, _Segment] = {}
        from torchstore_b200.epoch_board import reap_stale_segments

        reap_stale_segments()  # segments of killed jobs (their creators could not unlink them)

    def allocate(self, shape, dtype: torch.dtype) -> tuple[torch.Tensor, ShmDescriptor]:
        numel = 1
        for s in shape:
            numel *= s
        nbytes = max(numel * dtype.itemsize, 1)
        with _seq_lock:
            _seq[0] += 1
            name = f"/tsb200_{os.getpid()}_{_seq[0]}_{os.urandom(3).hex()}"
        ptr = _native.shm_create(name, nbytes)
        seg = self.segments[name] = _Segment(name, ptr, nbytes, owner=True)
        bisect.insort(self._starts, ptr)
        self._by_start[ptr] = seg
        seg.pin()
        stride, s = [], 1
        for e in reversed(shape):
            stride.append(s)
            s *= e
        stride = tuple(reversed(stride))
        tensor = _wrap(ptr, numel * dtype.itemsize, shape, stride, dtype)
        # the segment lives exactly as long as torch views of it do (stored tensor deleted / replaced
        # and every view gone -> unmap + unlink), like the HBM arena blocks
        self._storage_refs[name] = weakref.ref(tensor.untyped_storage(), lambda _r, _n=name: self._release(_n))
        return tensor, ShmDescriptor(name, nbytes, tuple(shape), stride, dtype)

    def _release(self, name: str) -> None:
        self._storage_refs.pop(name, None)
        seg = self.segments.pop(name, None)
        if seg is not None:
            self._forget_start(seg.ptr)
            seg.close()

    def _forget_start(self, ptr: int) -> None:
        self._by_start.pop(ptr, None)
        i = bisect.bisect_left(self._starts, ptr)
        if i < len(self._starts) and self._starts[i] == ptr:
            del self._starts[i]

    def describe(self, tensor: torch.Tensor) -> ShmDescriptor | None:
        """Descriptor of a stored tensor or of a view of one (None: not backed by our segments)."""
        ptr = tensor.data_ptr()
        i = bisect.bisect_right(self._starts, ptr) - 1
        if i < 0:
            return None
        seg = self._by_start[self._starts[i]]
        if not (seg.ptr <= ptr < seg.ptr + seg.nbytes):
            return None
        off = (ptr - seg.ptr) // tensor.element_size()
        return ShmDescriptor(seg.name, seg.nbytes, tuple(tensor.shape), tuple(tensor.stride()), tensor.dtype, off)

    def clear(self) -> None:
        self._storage_refs.clear()
        for seg in self.segments.values():
            seg.close()
        self.segments.clear()
        self._starts.clear()
        self._by_start.clear()


class HostClientCache(TransportCache):
    """Client side: attachments keyed by segment name (reference SharedMemoryCache, :210-260)."""

    def __init__(self) -> None:
        self.attached: dict[str, _Segment] = {}
        self._by_key: dict[str, set[str]] = {}

    def attach(self, desc: ShmDescriptor, key: str | None = None) -> _Segment:
        seg = self.attached.get(desc.name)
        if seg is None:
            ptr = _native.shm_attach(desc.name, desc.segment_bytes)
            seg = self.attached[desc.name] = _Segment(desc.name, ptr, desc.segment_bytes, owner=False)
        if key is not None:
            self._by_key.setdefault(key, set()).add(desc.name)
        return seg

    def view(self, desc: ShmDescriptor, key: str | None = None) -> torch.Tensor:
        seg = self.attach(desc, key)
        return _wrap(seg.ptr, seg.nbytes // desc.dtype.itemsize * desc.dtype.itemsize, desc.shape, desc.stride, desc.dtype,
                     desc.storage_offset)

    def delete(self, keys) -> None:
        """Drop the mappings of deleted keys (reference SharedMemoryCache.delete, :252-257)."""
        for key in keys:
            for name in self._by_key.pop(key, ()):
                seg = self.attached.pop(name, None)
                if seg is not None:
                    seg.close()

    def clear(self) -> None:
        for seg in self.attached.values():
            seg.close()
        self.attached.clear()
        self._by_key.clear()


def _host_move(pairs: list[tuple[torch.Tensor, torch.Tensor]]) -> None:
    """(src, dst) CPU tensor pairs of equal shape and dtype -> one threaded native call."""
    if not pairs:
        return
    for s, d in pairs:
        if s.dtype != d.dtype:
            raise AssertionError(f"{s.dtype} != {d.dtype}")
    rects, n = build_rects([(StridedMem.from_tensor(s), StridedMem.from_tensor(d)) for s, d in pairs])
    _native.host_copy_rects(rects, n, _COPY_THREADS)


class HostShmTransportBuffer(LandingBufferTransport):
    supports_strided_inplace = True  # the host mover writes strided destination rectangles directly

    # ---- volume memory: POSIX shm segments ------------------------------------------------------
    def _describe(self, ctx: "TransportContext", tensor: torch.Tensor) -> ShmDescriptor | None:
        return None if tensor.is_cuda else ctx.get(HostVolumeCache).describe(tensor)

    def _allocate(self, ctx: "TransportContext", shape: tuple, dtype: torch.dtype) -> tuple[torch.Tensor, ShmDescriptor]:
        return ctx.get(HostVolumeCache).allocate(shape, dtype)

    # ---- PUT ------------------------------------------------------------------------------------
    async def _post_handshake(self, handshake_results: list[Any], requests: list[Request]) -> None:
        cache: HostClientCache = self.storage_volume_ref.transport_context.get(HostClientCache)
        self._contexts = []
        host_pairs, devices, keep = [], set(), []
        for request, desc in zip(requests, handshake_results, strict=True):
            if request.is_object:
                self._contexts.append(EntryContext(objects=request.objects, use_rpc=True))
                continue
            tensor = request.tensor_val
            assert tensor is not None and desc is not None
            self._contexts.append(EntryContext(descriptor=desc))
            landing = cache.view(desc, request.key)
            if tensor.is_cuda:
                # D2H into the (pinned) segment, like the reference's shm_tensor.copy_(tensor) (:374)
                src = tensor if tensor.is_contiguous() else tensor.contiguous()
                seg = cache.attach(desc, request.key)
                seg.pin()
                dev = tensor.device.index
                staging_copy(dev, landing.data_ptr(), src.data_ptr(), desc.nbytes, _native.TSB_D2H)
                devices.add(dev)
                keep.append(src)
            else:
                host_pairs.append((tensor, landing))
        _host_move(host_pairs)
        for dev in devices:
            await wait_copy_stream(dev)  # polled from the loop, like the HBM transport

    # ---- GET ------------------------------------------------------------------------------------
    async def _handle_storage_volume_response(self, requests: list[Request], transport_buffer: "TransportBuffer") -> list[Any]:
        cache: HostClientCache = self.storage_volume_ref.transport_context.get(HostClientCache)
        results: list[Any] = [None] * len(requests)
        host_pairs, h2d, devices, keep = [], [], set(), []
        for i, (request, hctx) in enumerate(zip(requests, transport_buffer._contexts, strict=True)):
            dest = request.tensor_val
            if hctx.use_rpc:
                data = hctx.objects
                if isinstance(data, torch.Tensor) and dest is not None:
                    dest.copy_(data)
                    data = dest
                results[i] = data
                continue
            desc = hctx.descriptor
            assert desc is not None, f"No descriptor or data for key {request.key}"
            stored = cache.view(desc, request.key)
            gather = getattr(request, "_gather", None)
            if dest is None and gather is not None:
                dest = gather.view_for(request.tensor_slice, desc.dtype, torch.device("cpu"))
            if dest is None:
                # a private copy, never a live view of store memory (reference :478, MUTABLE_SHM=0)
                out = torch.empty(desc.shape, dtype=desc.dtype)
                host_pairs.append((stored, out))
                results[i] = out
                continue
            assert tuple(dest.shape) == tuple(desc.shape), f"{tuple(dest.shape)} != {tuple(desc.shape)}"
            if dest.is_cuda:
                h2d.append((stored, dest, desc))
            elif dest.dtype != desc.dtype:
                dest.copy_(stored)  # converting copy, like the reference's copy_
            else:
                host_pairs.append((stored, dest))
            results[i] = dest
        _host_move(host_pairs)
        for stored, dest, desc in h2d:
            dev = dest.device.index
            src = stored if stored.is_contiguous() else stored.contiguous()
            if dest.is_contiguous() and dest.dtype == desc.dtype:
                cache.attach(desc).pin()
                staging_copy(dev, dest.data_ptr(), src.data_ptr(), desc.nbytes, _native.TSB_H2D)
                devices.add(dev)
                keep.append(src)
            else:
                dest.copy_(src)
        for dev in devices:
            await wait_copy_stream(dev)
        return results

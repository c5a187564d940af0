"""Host-side planner: tensor layouts -> rectangle descriptors for the copy_rects kernel.

Two small value types carry everything the native layer needs, with no torch ops on the data:

* ``StridedMem``  -- (device pointer, shape, element strides, dtype, device): a tensor-shaped
  window onto HBM that may belong to another GPU/process.  ``sub(index)`` narrows it with pure
  pointer arithmetic, which is how a TensorSlice intersection becomes a source/destination
  rectangle without the reference's "read the whole shard, slice afterwards" step
  (reference direct_weight_sync.py:280-286).
* ``HbmDescriptor`` -- the picklable form (exported region + layout), the NVLink counterpart of
  ``SharedMemoryDescriptor`` (reference transport/shared_memory.py:99-164) and of the Monarch
  ``RDMABuffer`` handle (direct_weight_sync.py:143).
"""

from __future__ import annotations

import weakref
from dataclasses import dataclass
from typing import Sequence

import torch

from torchstore_b200 import _native

MAX_DIMS = _native.TSB_MAX_DIMS


@dataclass(frozen=True)
class StridedMem:
    ptr: int
    shape: tuple
    stride: tuple  # in elements
    dtype: torch.dtype
    device: int  # CUDA ordinal that physically holds the bytes; -1 for host memory (tests)

    @classmethod
    def from_tensor(cls, t: torch.Tensor) -> "StridedMem":
        dev = t.device.index if t.is_cuda else -1
        if t.is_cuda and dev is None:
            dev = torch.cuda.current_device()
        return cls(t.data_ptr(), tuple(t.shape), tuple(t.stride()), t.dtype, dev)

    @property
    def itemsize(self) -> int:
        return self.dtype.itemsize

    @property
    def numel(self) -> int:
        n = 1
        for s in self.shape:
            n *= s
        return n

    def sub(self, index: Sequence[slice]) -> "StridedMem":
        """Window ``self[index]`` for unit-step slices (one per dimension)."""
        if len(index) != len(self.shape):
            raise ValueError(f"index rank {len(index)} != tensor rank {len(self.shape)}")
        off = 0
        shape = []
        for sl, extent, st in zip(index, self.shape, self.stride):
            start, stop, step = sl.indices(extent)
            if step != 1:
                raise ValueError("only unit-step slices describe a rectangle")
            off += start * st
            shape.append(max(0, stop - start))
        return StridedMem(self.ptr + off * self.itemsize, tuple(shape), self.stride, self.dtype, self.device)

    def is_contiguous(self) -> bool:
        expected = 1
        for extent, st in zip(reversed(self.shape), reversed(self.stride)):
            if extent == 1:
                continue
            if st != expected:
                return False
            expected *= extent
        return True

    def flat_bytes(self) -> "StridedMem":
        """1-D uint8 alias of a contiguous window."""
        if not self.is_contiguous():
            raise ValueError("flat_bytes needs a contiguous window")
        return StridedMem(self.ptr, (self.numel * self.itemsize,), (1,), torch.uint8, self.device)


def _collapse(shape, sstride, dstride):
    """Merge adjacent dims that are jointly contiguous in BOTH layouts; drop unit dims."""
    dims = [(e, ss, ds) for e, ss, ds in zip(shape, sstride, dstride) if e != 1]
    out: list[tuple[int, int, int]] = []
    for e, ss, ds in dims:
        if out:
            pe, pss, pds = out[-1]
            if pss == ss * e and pds == ds * e:
                out[-1] = (pe * e, ss, ds)
                continue
        out.append((e, ss, ds))
    return out


_FLOATS = (torch.bfloat16, torch.float16, torch.float32)


def fill_rect(rect: "_native.Rect", src: StridedMem, dst: StridedMem, quantise: bool = False,
              dequantise: bool = False) -> bool:
    """Fill a tsb_rect_t moving window ``src`` onto window ``dst`` (same shape; dtypes may differ
    when the pair is a supported cast).  Returns False for an empty window (nothing to move).
    ``quantise``: the window feeds a quantising plan, where a bf16/f16/f32 -> int8 window is TSB_I8 on its
    destination side; ``dequantise``: a dequantising plan, where an int8 -> bf16/f16/f32 window is TSB_I8 on
    its source side."""
    if tuple(src.shape) != tuple(dst.shape):
        raise ValueError(f"source window {src.shape} and destination window {dst.shape} differ")
    int8 = quantise and dst.dtype == torch.int8 and src.dtype in _FLOATS
    int8_src = dequantise and src.dtype == torch.int8 and dst.dtype in _FLOATS
    if src.dtype != dst.dtype and not int8 and not int8_src and not _native.cast_supported(src.dtype, dst.dtype):
        raise NotImplementedError(f"no fused cast kernel for {src.dtype} -> {dst.dtype}")
    if any(e == 0 for e in src.shape):
        return False
    sb, db = src.itemsize, dst.itemsize
    dims = _collapse(src.shape, [s * sb for s in src.stride], [s * db for s in dst.stride])
    if not dims:
        dims = [(1, sb, db)]
    if len(dims) > MAX_DIMS:
        raise NotImplementedError(f"rectangle has {len(dims)} non-mergeable dims (> {MAX_DIMS})")
    rect.src = src.ptr
    rect.dst = dst.ptr
    rect.ndim = len(dims)
    for i, (e, ss, ds) in enumerate(dims):
        rect.extent[i] = e
        rect.src_stride[i] = ss
        rect.dst_stride[i] = ds
    for i in range(len(dims), MAX_DIMS):
        rect.extent[i] = 1
        rect.src_stride[i] = 0
        rect.dst_stride[i] = 0
    if src.dtype == dst.dtype:
        code = _native.dtype_code(src.dtype)
        if src.itemsize == 16:  # complex128: two 8-byte words per element
            raise NotImplementedError("16-byte elements are not supported")
        rect.src_dtype = rect.dst_dtype = code
    else:
        rect.src_dtype = _native.TSB_I8 if int8_src else _native.cast_code(src.dtype)
        rect.dst_dtype = _native.TSB_I8 if int8 else _native.cast_code(dst.dtype)
    rect.src_device = src.device
    return True


def build_rects(pairs: Sequence[tuple[StridedMem, StridedMem]], quantise: bool = False, dequantise: bool = False):
    """(src, dst) windows -> (ctypes array of tsb_rect_t, count).  Empty windows are skipped.  ``quantise``,
    ``dequantise``: as for :func:`fill_rect`."""
    arr = _native.make_rect_array(max(1, len(pairs)))
    n = 0
    for src, dst in pairs:
        if fill_rect(arr[n], src, dst, quantise, dequantise):
            n += 1
    return arr, n


def build_transpose_rects(pairs: Sequence[tuple[StridedMem, StridedMem]]):
    """(src, dst) windows of transposed packed parts -> (ctypes array of tsb_rect_t, count), for
    tsb_transpose_plan_create.  Unlike :func:`build_rects` the last two dims stay as they are, unit extents included:
    they are the transposed pair (destination contiguous along dim -1, source along dim -2).  The outer dims lose
    their unit extents.  Empty windows are skipped."""
    arr = _native.make_rect_array(max(1, len(pairs)))
    n = 0
    for src, dst in pairs:
        if tuple(src.shape) != tuple(dst.shape):
            raise ValueError(f"source window {src.shape} and destination window {dst.shape} differ")
        if src.dtype != dst.dtype and not _native.cast_supported(src.dtype, dst.dtype):
            raise NotImplementedError(f"no fused cast kernel for {src.dtype} -> {dst.dtype}")
        if len(src.shape) < 2 or any(e == 0 for e in src.shape):
            continue
        sb, db = src.itemsize, dst.itemsize
        outer = [(e, ss * sb, ds * db) for e, ss, ds in zip(src.shape[:-2], src.stride[:-2], dst.stride[:-2]) if e != 1]
        dims = outer + [(e, ss * sb, ds * db) for e, ss, ds in zip(src.shape[-2:], src.stride[-2:], dst.stride[-2:])]
        if len(dims) > MAX_DIMS:
            raise NotImplementedError(f"rectangle has {len(dims)} dims (> {MAX_DIMS})")
        rect = arr[n]
        rect.src, rect.dst, rect.ndim = src.ptr, dst.ptr, len(dims)
        for i in range(MAX_DIMS):
            rect.extent[i], rect.src_stride[i], rect.dst_stride[i] = dims[i] if i < len(dims) else (1, 0, 0)
        if src.dtype == dst.dtype:
            rect.src_dtype = rect.dst_dtype = _native.dtype_code(src.dtype)
        else:
            rect.src_dtype, rect.dst_dtype = _native.cast_code(src.dtype), _native.cast_code(dst.dtype)
        rect.src_device = src.device
        n += 1
    return arr, n


# ------------------------------------------------------------------------------------------------
# picklable handle
# ------------------------------------------------------------------------------------------------
def _span_elems(shape, stride) -> int:
    """Elements between the first and one-past-the-last element touched (non-negative strides)."""
    if any(e == 0 for e in shape):
        return 0
    return sum((e - 1) * st for e, st in zip(shape, stride)) + 1


class _ExportCache:
    """Exporter-side registration cache: (data_ptr, nbytes) -> exported region, evicted when the
    tensor's storage dies -- the counterpart of the reference's RdmaMemoryCache
    (transport/torchcomms/cache.py:150-186: keyed on (data_ptr, nbytes), weakref on
    ``untyped_storage()``).  Saves the driver round trips (cuMemGetAddressRange, cudaIpcGetMemHandle)
    on every get of a stored tensor and on every handle re-publication."""

    def __init__(self) -> None:
        self._regions: dict[tuple[int, int], tuple[bytes, int]] = {}
        self._storage_refs: dict[tuple[int, int], weakref.ref] = {}
        self.hits = self.misses = self.evictions = 0

    def export(self, t: torch.Tensor, nbytes: int) -> tuple[bytes, int]:
        # torch reports a null data pointer for a tensor without elements (an empty shard, or an empty
        # window of a stored tensor); its storage still has an address to describe, and no copy reads it
        ptr = t.data_ptr() or t.untyped_storage().data_ptr()
        key = (ptr, nbytes)
        hit = self._regions.get(key)
        if hit is not None:
            self.hits += 1
            return hit
        self.misses += 1
        region = _native.export_region(ptr, nbytes)
        entry = (_native.region_to_bytes(region), int(region.device))
        try:
            ref = weakref.ref(t.untyped_storage(), lambda _r, _k=key: self._evict(_k))
        except Exception:  # storage not weak-referenceable: do not cache what cannot be invalidated
            return entry
        self._regions[key] = entry
        self._storage_refs[key] = ref
        return entry

    def _evict(self, key) -> None:
        if self._regions.pop(key, None) is not None:
            self.evictions += 1
        self._storage_refs.pop(key, None)

    def clear(self) -> None:
        self._regions.clear()
        self._storage_refs.clear()


export_cache = _ExportCache()


@dataclass
class HbmDescriptor:
    """Where a tensor lives in some GPU's HBM, in a form that survives pickling."""

    region: bytes  # tsb_region_t covering the tensor's bytes
    shape: tuple
    stride: tuple
    dtype: torch.dtype
    device: int  # exporter's CUDA ordinal

    @classmethod
    def from_tensor(cls, t: torch.Tensor) -> "HbmDescriptor":
        if not t.is_cuda:
            raise ValueError("HbmDescriptor.from_tensor needs a CUDA tensor (there is no host data plane)")
        if any(st < 0 for st in t.stride()):
            raise ValueError("negative strides are not supported")
        nbytes = _span_elems(t.shape, t.stride()) * t.element_size()
        raw, device = export_cache.export(t, max(nbytes, 1))
        return cls(raw, tuple(t.shape), tuple(t.stride()), t.dtype, device)

    @property
    def nbytes(self) -> int:
        n = self.dtype.itemsize
        for s in self.shape:
            n *= s
        return n

    def resolve(self, device: int) -> StridedMem:
        """Map into this process (cached natively) and return a window kernels on ``device`` can read."""
        region = _native.region_from_bytes(self.region)
        ptr = _native.import_region(region, device)
        return StridedMem(ptr, tuple(self.shape), tuple(self.stride), self.dtype, self.device)

    def release(self) -> None:
        _native.release_region(_native.region_from_bytes(self.region))

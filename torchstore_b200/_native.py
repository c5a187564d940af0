"""ctypes binding of libtstore_b200.so (see include/tstore_b200.h).

There is no fallback: if the library is missing or a call fails, a Python exception is raised
with the library's own message (status-int convention of the reference's native transports,
transport/torchcomms/buffer.py:238-239).
"""

from __future__ import annotations

import ctypes as C
import os
import threading

import torch

from torchstore_b200._build import LIB_PATH

TSB_MAX_DIMS = 6
TSB_ABI_VERSION = 2

TSB_OK, TSB_ERR_INVALID, TSB_ERR_CUDA, TSB_ERR_UNSUPPORTED, TSB_ERR_NOMEM, TSB_ERR_NOTFOUND = range(6)

TSB_U8, TSB_U16, TSB_U32, TSB_U64, TSB_F16, TSB_BF16, TSB_F32, TSB_F64 = range(8)
TSB_H2D, TSB_D2H, TSB_D2D = 1, 2, 3
TSB_PLAN_DEFAULT, TSB_PLAN_NO_INTERLEAVE = 0, 1


class TsbError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"tstore_b200 native error {code}: {msg}")
        self.code = code


class Region(C.Structure):
    """tsb_region_t -- picklable via bytes(region)."""

    _fields_ = [
        ("ipc_handle", C.c_uint8 * 64),
        ("offset", C.c_uint64),
        ("nbytes", C.c_uint64),
        ("alloc_bytes", C.c_uint64),
        ("local_ptr", C.c_uint64),
        ("device", C.c_int32),
        ("pid", C.c_int32),
        ("boot_id", C.c_uint64),
        ("epoch", C.c_uint64),
    ]


class Rect(C.Structure):
    """tsb_rect_t"""

    _fields_ = [
        ("src", C.c_uint64),
        ("dst", C.c_uint64),
        ("extent", C.c_int64 * TSB_MAX_DIMS),
        ("src_stride", C.c_int64 * TSB_MAX_DIMS),
        ("dst_stride", C.c_int64 * TSB_MAX_DIMS),
        ("ndim", C.c_uint32),
        ("src_dtype", C.c_uint32),
        ("dst_dtype", C.c_uint32),
        ("src_device", C.c_int32),
    ]


class PlanInfo(C.Structure):
    _fields_ = [
        ("num_rects", C.c_uint64),
        ("num_tiles", C.c_uint64),
        ("payload_bytes", C.c_uint64),
        ("src_bytes", C.c_uint64),
        ("remote_src_bytes", C.c_uint64),
        ("num_link_tiles", C.c_uint64),
        ("link_bytes", C.c_uint64),
        ("grid", C.c_uint32),
        ("block", C.c_uint32),
        ("tile_bytes", C.c_uint32),
        ("num_vector_rects", C.c_uint32),
        ("link_tile_bytes", C.c_uint32),
        ("link_stages", C.c_uint32),
    ]

    def as_dict(self) -> dict:
        return {name: int(getattr(self, name)) for name, _ in self._fields_}


class ArenaStats(C.Structure):
    _fields_ = [
        ("capacity", C.c_uint64),
        ("in_use", C.c_uint64),
        ("high_water", C.c_uint64),
        ("num_blocks", C.c_uint64),
        ("base", C.c_uint64),
    ]


# every symbol include/tstore_b200.h declares: name -> (restype, argtypes)
_vp = C.c_void_p
_SIGNATURES = {
    "tsb_abi_version": (C.c_int, []),
    "tsb_last_error": (C.c_char_p, []),
    "tsb_init": (C.c_int, []),
    "tsb_shutdown": (C.c_int, []),
    "tsb_device_count": (C.c_int, [C.POINTER(C.c_int)]),
    "tsb_enable_peer_access": (C.c_int, [C.c_int, C.c_int]),
    "tsb_launch_count": (C.c_uint64, []),
    "tsb_export_region": (C.c_int, [_vp, C.c_uint64, C.POINTER(Region)]),
    "tsb_import_region": (C.c_int, [C.POINTER(Region), C.c_int, C.POINTER(_vp)]),
    "tsb_release_region": (C.c_int, [C.POINTER(Region)]),
    "tsb_release_all": (C.c_int, []),
    "tsb_import_stats": (C.c_int, [C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "tsb_cast_supported": (C.c_int, [C.c_uint32, C.c_uint32]),
    "tsb_plan_create": (C.c_int, [C.c_int, C.POINTER(Rect), C.c_uint64, C.c_uint32, C.POINTER(C.c_uint64)]),
    "tsb_plan_info": (C.c_int, [C.c_uint64, C.POINTER(PlanInfo)]),
    "tsb_plan_run": (C.c_int, [C.c_uint64, _vp]),
    "tsb_plan_launch": (C.c_int, [C.c_uint64, _vp]),
    "tsb_plan_launch_flags": (C.c_int, [C.c_uint64, _vp, C.c_uint32]),
    "tsb_plan_poll": (C.c_int, [C.c_uint64, C.POINTER(C.c_int)]),
    "tsb_plan_wait": (C.c_int, [C.c_uint64]),
    "tsb_plan_elapsed_ms": (C.c_int, [C.c_uint64, C.POINTER(C.c_float)]),
    "tsb_plan_destroy": (C.c_int, [C.c_uint64]),
    "tsb_pool_stats": (C.c_int, [C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]),
    "tsb_plan_compile_host": (
        C.c_int,
        [C.c_int, C.POINTER(Rect), C.c_uint64, C.c_uint32, C.c_uint32, _vp, C.c_uint64, C.POINTER(C.c_uint64),
         _vp, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(PlanInfo)],
    ),
    "tsb_copy_rects": (C.c_int, [C.c_int, C.POINTER(Rect), C.c_uint64, C.c_uint32, _vp]),
    "tsb_stream_create": (C.c_int, [C.c_int, C.POINTER(_vp)]),
    "tsb_stream_destroy": (C.c_int, [_vp]),
    "tsb_stream_sync": (C.c_int, [C.c_int, _vp]),
    "tsb_copy_stream": (C.c_int, [C.c_int, C.POINTER(_vp)]),
    "tsb_event_create": (C.c_int, [C.c_int, C.c_int, C.POINTER(_vp)]),
    "tsb_event_record": (C.c_int, [_vp, C.c_int, _vp]),
    "tsb_stream_wait_event": (C.c_int, [C.c_int, _vp, _vp]),
    "tsb_event_query": (C.c_int, [_vp, C.POINTER(C.c_int)]),
    "tsb_event_sync": (C.c_int, [_vp]),
    "tsb_event_elapsed_ms": (C.c_int, [_vp, _vp, C.POINTER(C.c_float)]),
    "tsb_event_destroy": (C.c_int, [_vp]),
    "tsb_arena_create": (C.c_int, [C.c_int, C.c_uint64, C.POINTER(C.c_uint64)]),
    "tsb_arena_alloc": (C.c_int, [C.c_uint64, C.c_uint64, C.c_uint64, C.POINTER(_vp)]),
    "tsb_arena_free": (C.c_int, [C.c_uint64, _vp]),
    "tsb_arena_stats": (C.c_int, [C.c_uint64, C.POINTER(ArenaStats)]),
    "tsb_arena_destroy": (C.c_int, [C.c_uint64]),
    "tsb_host_alloc": (C.c_int, [C.c_uint64, C.POINTER(_vp)]),
    "tsb_host_free": (C.c_int, [_vp]),
    "tsb_host_register": (C.c_int, [_vp, C.c_uint64]),
    "tsb_host_unregister": (C.c_int, [_vp]),
    "tsb_memcpy_async": (C.c_int, [C.c_int, _vp, _vp, C.c_uint64, C.c_int, _vp]),
    "tsb_shm_create": (C.c_int, [C.c_char_p, C.c_uint64, C.POINTER(_vp)]),
    "tsb_shm_attach": (C.c_int, [C.c_char_p, C.c_uint64, C.POINTER(_vp)]),
    "tsb_shm_detach": (C.c_int, [_vp, C.c_uint64]),
    "tsb_shm_unlink": (C.c_int, [C.c_char_p]),
    "tsb_host_copy_rects": (C.c_int, [C.POINTER(Rect), C.c_uint64, C.c_uint32]),
}

EXPORTED_SYMBOLS = tuple(_SIGNATURES)

_lib = None
_lib_lock = threading.Lock()


def lib() -> C.CDLL:
    """Load libtstore_b200.so (once).  Raises if it has not been built -- never falls back."""
    global _lib
    if _lib is not None:
        return _lib
    with _lib_lock:
        if _lib is not None:
            return _lib
        path = os.environ.get("TSTORE_B200_LIB", LIB_PATH)
        if not os.path.exists(path):
            raise RuntimeError(
                f"libtstore_b200.so not found at {path}. Build it with "
                "`python -c 'import __graft_entry__ as g; g.build()'` (needs nvcc). "
                "torchstore_b200 has no CPU or PyTorch fallback for its data plane."
            )
        handle = C.CDLL(path)
        for name, (restype, argtypes) in _SIGNATURES.items():
            fn = getattr(handle, name)  # AttributeError if the header and the library diverge
            fn.restype = restype
            fn.argtypes = argtypes
        if handle.tsb_abi_version() != TSB_ABI_VERSION:
            raise RuntimeError("libtstore_b200.so ABI version mismatch; rebuild it")
        _lib = handle
    return _lib


def check(status: int) -> None:
    if status != TSB_OK:
        msg = lib().tsb_last_error().decode(errors="replace")
        raise TsbError(status, msg)


# ------------------------------------------------------------------------------------------------
# dtype mapping
# ------------------------------------------------------------------------------------------------
_FLOAT_CODES = {
    torch.float16: TSB_F16,
    torch.bfloat16: TSB_BF16,
    torch.float32: TSB_F32,
    torch.float64: TSB_F64,
}
_OPAQUE_BY_SIZE = {1: TSB_U8, 2: TSB_U16, 4: TSB_U32, 8: TSB_U64}


def dtype_code(dtype: torch.dtype) -> int:
    """TSB_* code for a torch dtype.  Non-float dtypes map to opaque fixed-width codes, which can
    only be byte-copied (never cast)."""
    code = _FLOAT_CODES.get(dtype)
    if code is not None:
        return code
    size = dtype.itemsize
    if size in _OPAQUE_BY_SIZE:
        return _OPAQUE_BY_SIZE[size]
    if size == 16:  # complex128: moved as pairs of 8-byte words by the caller
        return TSB_U64
    raise TypeError(f"unsupported dtype {dtype}")


def cast_supported(src: torch.dtype, dst: torch.dtype) -> bool:
    if src == dst:
        return True
    if src not in _FLOAT_CODES or dst not in _FLOAT_CODES:
        return False
    return bool(lib().tsb_cast_supported(_FLOAT_CODES[src], _FLOAT_CODES[dst]))


# ------------------------------------------------------------------------------------------------
# thin helpers
# ------------------------------------------------------------------------------------------------
def init() -> None:
    check(lib().tsb_init())


def device_count() -> int:
    n = C.c_int(0)
    check(lib().tsb_device_count(C.byref(n)))
    return n.value


def launch_count() -> int:
    return int(lib().tsb_launch_count())


def enable_peer_access(device: int, peer: int) -> None:
    check(lib().tsb_enable_peer_access(device, peer))


def export_region(ptr: int, nbytes: int) -> Region:
    reg = Region()
    check(lib().tsb_export_region(C.c_void_p(ptr), nbytes, C.byref(reg)))
    return reg


def import_region(region: Region, device: int) -> int:
    out = C.c_void_p()
    check(lib().tsb_import_region(C.byref(region), device, C.byref(out)))
    return int(out.value)


def release_region(region: Region) -> None:
    check(lib().tsb_release_region(C.byref(region)))


def release_all() -> None:
    check(lib().tsb_release_all())


def import_stats() -> dict:
    live, stale = C.c_uint64(0), C.c_uint64(0)
    check(lib().tsb_import_stats(C.byref(live), C.byref(stale)))
    return {"live": live.value, "stale_evictions": stale.value}


def region_to_bytes(region: Region) -> bytes:
    return bytes(region)


def region_from_bytes(raw: bytes) -> Region:
    if len(raw) != C.sizeof(Region):
        raise ValueError("bad region blob")
    return Region.from_buffer_copy(raw)


def make_rect_array(n: int):
    return (Rect * n)()


def plan_create(device: int, rects, n: int, flags: int = TSB_PLAN_DEFAULT) -> int:
    out = C.c_uint64(0)
    check(lib().tsb_plan_create(device, rects, n, flags, C.byref(out)))
    return int(out.value)


def plan_info(plan: int) -> PlanInfo:
    info = PlanInfo()
    check(lib().tsb_plan_info(plan, C.byref(info)))
    return info


def plan_run(plan: int, stream: int | None = None) -> None:
    check(lib().tsb_plan_run(plan, C.c_void_p(stream) if stream else None))


TSB_LAUNCH_NO_FENCE_OUT = 1


def plan_launch(plan: int, caller_stream: int | None = None, fence_out: bool = True) -> None:
    """fence-in, start event, kernel, done event, fence-out: one native call per sync.
    ``fence_out=False``: the caller's stream is not made to wait for the copy (overlapping puts)."""
    check(lib().tsb_plan_launch_flags(plan, C.c_void_p(caller_stream) if caller_stream else None,
                                      0 if fence_out else TSB_LAUNCH_NO_FENCE_OUT))


def plan_poll(plan: int) -> bool:
    done = C.c_int(0)  # per call: ctypes drops the GIL, so threads may poll concurrently
    check(lib().tsb_plan_poll(plan, C.byref(done)))
    return bool(done.value)


def plan_wait(plan: int) -> None:
    check(lib().tsb_plan_wait(plan))


def plan_elapsed_ms(plan: int) -> float:
    ms = C.c_float(0)
    check(lib().tsb_plan_elapsed_ms(plan, C.byref(ms)))
    return float(ms.value)


def plan_destroy(plan: int) -> None:
    check(lib().tsb_plan_destroy(plan))


def pool_stats() -> dict:
    b, a, r = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
    check(lib().tsb_pool_stats(C.byref(b), C.byref(a), C.byref(r)))
    return {"blocks": b.value, "allocs": a.value, "reuses": r.value}


def copy_rects(device: int, rects, n: int, flags: int = TSB_PLAN_DEFAULT, stream: int | None = None) -> None:
    check(lib().tsb_copy_rects(device, rects, n, flags, C.c_void_p(stream) if stream else None))


def plan_compile_host(device: int, rects, n: int, flags: int = 0, tile_units: int = 0):
    """Host-only plan compilation -> (rect_table_bytes, tile_array[(rect, tile_in_rect)], PlanInfo)."""
    import numpy as np

    n_rects = C.c_uint64(0)
    n_tiles = C.c_uint64(0)
    info = PlanInfo()
    L = lib()
    check(L.tsb_plan_compile_host(device, rects, n, flags, tile_units, None, 0, C.byref(n_rects), None, 0,
                                  C.byref(n_tiles), C.byref(info)))
    rect_buf = np.zeros(max(1, n_rects.value) * 192, dtype=np.uint8)
    tile_buf = np.zeros((max(1, n_tiles.value), 2), dtype=np.uint32)
    check(L.tsb_plan_compile_host(device, rects, n, flags, tile_units, rect_buf.ctypes.data, n_rects.value,
                                  C.byref(n_rects), tile_buf.ctypes.data, n_tiles.value, C.byref(n_tiles),
                                  C.byref(info)))
    return rect_buf[: n_rects.value * 192], tile_buf[: n_tiles.value], info


CUDA_STREAM_LEGACY = 0x1  # cudaStreamLegacy: an explicit handle for the default stream


def torch_stream(device: int | None = None) -> int:
    """cudaStream_t of torch's current stream as a value the C-ABI can take.  torch reports the
    legacy default stream as 0, which the ABI reserves for "the library's copy stream"; map it to
    the explicit cudaStreamLegacy handle."""
    h = torch.cuda.current_stream(device).cuda_stream
    return h if h else CUDA_STREAM_LEGACY


def copy_stream(device: int) -> int:
    out = C.c_void_p()
    check(lib().tsb_copy_stream(device, C.byref(out)))
    return int(out.value)


def stream_sync(device: int, stream: int | None = None) -> None:
    check(lib().tsb_stream_sync(device, C.c_void_p(stream) if stream else None))


class Event:
    """cudaEvent_t owned by the library."""

    def __init__(self, device: int, timing: bool = False):
        self.device = device
        out = C.c_void_p()
        check(lib().tsb_event_create(device, 1 if timing else 0, C.byref(out)))
        self.handle = out.value

    def record(self, stream: int | None = None) -> "Event":
        check(lib().tsb_event_record(C.c_void_p(self.handle), self.device, C.c_void_p(stream) if stream else None))
        return self

    def wait_on(self, device: int, stream: int | None = None) -> None:
        """Make `stream` (NULL: the copy stream of `device`) wait for this event."""
        check(lib().tsb_stream_wait_event(device, C.c_void_p(stream) if stream else None, C.c_void_p(self.handle)))

    def query(self) -> bool:
        done = C.c_int(0)
        check(lib().tsb_event_query(C.c_void_p(self.handle), C.byref(done)))
        return bool(done.value)

    def synchronize(self) -> None:
        check(lib().tsb_event_sync(C.c_void_p(self.handle)))

    def elapsed_ms(self, later: "Event") -> float:
        ms = C.c_float(0)
        check(lib().tsb_event_elapsed_ms(C.c_void_p(self.handle), C.c_void_p(later.handle), C.byref(ms)))
        return float(ms.value)

    def close(self) -> None:
        if self.handle:
            lib().tsb_event_destroy(C.c_void_p(self.handle))
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def arena_create(device: int, capacity: int) -> int:
    out = C.c_uint64(0)
    check(lib().tsb_arena_create(device, capacity, C.byref(out)))
    return int(out.value)


def arena_alloc(arena: int, nbytes: int, align: int = 256) -> int:
    out = C.c_void_p()
    check(lib().tsb_arena_alloc(arena, nbytes, align, C.byref(out)))
    return int(out.value)


def arena_free(arena: int, ptr: int) -> None:
    check(lib().tsb_arena_free(arena, C.c_void_p(ptr)))


def arena_stats(arena: int) -> ArenaStats:
    st = ArenaStats()
    check(lib().tsb_arena_stats(arena, C.byref(st)))
    return st


def arena_destroy(arena: int) -> None:
    check(lib().tsb_arena_destroy(arena))


def host_alloc(nbytes: int) -> int:
    out = C.c_void_p()
    check(lib().tsb_host_alloc(nbytes, C.byref(out)))
    return int(out.value)


def host_free(ptr: int) -> None:
    check(lib().tsb_host_free(C.c_void_p(ptr)))


def host_register(ptr: int, nbytes: int) -> None:
    check(lib().tsb_host_register(C.c_void_p(ptr), nbytes))


def host_unregister(ptr: int) -> None:
    check(lib().tsb_host_unregister(C.c_void_p(ptr)))


def memcpy_async(device: int, dst: int, src: int, nbytes: int, kind: int, stream: int | None = None) -> None:
    check(lib().tsb_memcpy_async(device, C.c_void_p(dst), C.c_void_p(src), nbytes, kind,
                                 C.c_void_p(stream) if stream else None))


# ---- host tier (no CUDA device needed) -----------------------------------------------------------
def shm_create(name: str, nbytes: int) -> int:
    out = C.c_void_p()
    check(lib().tsb_shm_create(name.encode(), nbytes, C.byref(out)))
    return int(out.value)


def shm_attach(name: str, nbytes: int) -> int:
    out = C.c_void_p()
    check(lib().tsb_shm_attach(name.encode(), nbytes, C.byref(out)))
    return int(out.value)


def shm_detach(ptr: int, nbytes: int) -> None:
    check(lib().tsb_shm_detach(C.c_void_p(ptr), nbytes))


def shm_unlink(name: str) -> None:
    check(lib().tsb_shm_unlink(name.encode()))


def host_copy_rects(rects, n: int, threads: int = 1) -> None:
    check(lib().tsb_host_copy_rects(rects, n, threads))

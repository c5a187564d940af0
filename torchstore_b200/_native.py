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
TSB_ABI_VERSION = 9

TSB_OK, TSB_ERR_INVALID, TSB_ERR_CUDA, TSB_ERR_UNSUPPORTED, TSB_ERR_NOMEM, TSB_ERR_NOTFOUND = range(6)

TSB_U8, TSB_U16, TSB_U32, TSB_U64, TSB_F16, TSB_BF16, TSB_F32, TSB_F64, TSB_F8E4M3, TSB_F8E5M2 = range(10)
TSB_H2D, TSB_D2H, TSB_D2D = 1, 2, 3
TSB_PLAN_DEFAULT, TSB_PLAN_NO_INTERLEAVE = 0, 1
TSB_QUANT_UE8M0 = 1  # flags of the quantising plan calls: power-of-two scales
TSB_I8 = 10  # int8: dst_dtype of a quantising pull's rects (tsb_block_fp8_*, tsb_scaled_fp8_*), src_dtype of a
# dequantising pull's (tsb_dequant_fp8_*), dst_dtype of tsb_source_quant_*_as


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


class BqTarget(C.Structure):
    """tsb_bq_target_t: one block-scaled fp8 destination."""

    _fields_ = [
        ("dst", C.c_uint64),
        ("scale_inv", C.c_uint64),
        ("batch", C.c_uint64),
        ("rows", C.c_uint64),
        ("cols", C.c_uint64),
    ]


TSB_SCALE_PER_CHANNEL, TSB_SCALE_PER_TENSOR = 1, 2


class SqTarget(C.Structure):
    """tsb_sq_target_t: one per-channel or per-tensor scaled fp8 destination."""

    _fields_ = [
        ("dst", C.c_uint64),
        ("scale_inv", C.c_uint64),
        ("batch", C.c_uint64),
        ("rows", C.c_uint64),
        ("cols", C.c_uint64),
        ("granularity", C.c_uint32),
        ("pad", C.c_uint32),
    ]


TSB_SCALE_PER_BLOCK = 3


class DqSource(C.Structure):
    """tsb_dq_source_t: one block-, channel- or tensor-scaled fp8 source shard of a dequantising pull."""

    _fields_ = [
        ("src", C.c_uint64),
        ("scale", C.c_uint64),
        ("batch", C.c_uint64),
        ("rows", C.c_uint64),
        ("cols", C.c_uint64),
        ("row0", C.c_uint64),
        ("col0", C.c_uint64),
        ("granularity", C.c_uint32),
        ("pad", C.c_uint32),
    ]


class SourceQuantTarget(C.Structure):
    """tsb_source_quant_target_t: one bf16/f16/f32 shard quantised into scaled fp8 staging on its own device."""

    _fields_ = [
        ("src", C.c_uint64),
        ("dst", C.c_uint64),
        ("scale_inv", C.c_uint64),
        ("batch", C.c_uint64),
        ("rows", C.c_uint64),
        ("cols", C.c_uint64),
        ("row0", C.c_uint64),
        ("col0", C.c_uint64),
        ("src_dtype", C.c_uint32),
        ("granularity", C.c_uint32),
    ]


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
    "tsb_block_fp8_plan_create": (
        C.c_int, [C.c_int, C.POINTER(Rect), C.c_uint64, C.POINTER(BqTarget), C.c_uint64, C.c_uint32, C.POINTER(C.c_uint64)],
    ),
    "tsb_block_fp8_compile_host": (
        C.c_int,
        [C.c_int, C.POINTER(Rect), C.c_uint64, C.POINTER(BqTarget), C.c_uint64, C.c_uint32, _vp, C.c_uint64,
         C.POINTER(C.c_uint64), _vp, C.c_uint64, C.POINTER(C.c_uint64)],
    ),
    "tsb_scaled_fp8_plan_create": (
        C.c_int, [C.c_int, C.POINTER(Rect), C.c_uint64, C.POINTER(SqTarget), C.c_uint64, C.c_uint32, C.POINTER(C.c_uint64)],
    ),
    "tsb_scaled_fp8_compile_host": (
        C.c_int,
        [C.c_int, C.POINTER(Rect), C.c_uint64, C.POINTER(SqTarget), C.c_uint64, C.c_uint32, _vp, C.c_uint64,
         C.POINTER(C.c_uint64), _vp, C.c_uint64, C.POINTER(C.c_uint64), _vp, C.c_uint64, C.POINTER(C.c_uint64),
         C.POINTER(C.c_uint64)],
    ),
    "tsb_dequant_fp8_plan_create": (
        C.c_int, [C.c_int, C.POINTER(Rect), C.c_uint64, C.POINTER(DqSource), C.c_uint64, C.c_uint32, C.POINTER(C.c_uint64)],
    ),
    "tsb_dequant_fp8_compile_host": (
        C.c_int,
        [C.c_int, C.POINTER(Rect), C.c_uint64, C.POINTER(DqSource), C.c_uint64, C.c_uint32, _vp, C.c_uint64,
         C.POINTER(C.c_uint64)],
    ),
    "tsb_requant_fp8_plan_create": (
        C.c_int,
        [C.c_int, C.POINTER(Rect), C.c_uint64, C.POINTER(DqSource), C.c_uint64, C.POINTER(SqTarget), C.c_uint64, C.c_uint32,
         C.POINTER(C.c_uint64)],
    ),
    "tsb_requant_fp8_compile_host": (
        C.c_int,
        [C.c_int, C.POINTER(Rect), C.c_uint64, C.POINTER(DqSource), C.c_uint64, C.POINTER(SqTarget), C.c_uint64, C.c_uint32,
         _vp, C.c_uint64, C.POINTER(C.c_uint64), _vp, C.c_uint64, C.POINTER(C.c_uint64), _vp, C.c_uint64,
         C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)],
    ),
    "tsb_source_quant_plan_create": (
        C.c_int, [C.c_int, C.POINTER(SourceQuantTarget), C.c_uint64, C.c_uint32, C.POINTER(C.c_uint64)],
    ),
    "tsb_source_quant_compile_host": (
        C.c_int,
        [C.c_int, C.POINTER(SourceQuantTarget), C.c_uint64, C.c_uint32, _vp, C.c_uint64, C.POINTER(C.c_uint64), _vp,
         C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)],
    ),
    "tsb_source_quant_plan_create_as": (
        C.c_int, [C.c_int, C.POINTER(SourceQuantTarget), C.c_uint64, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint64)],
    ),
    "tsb_source_quant_compile_host_as": (
        C.c_int,
        [C.c_int, C.POINTER(SourceQuantTarget), C.c_uint64, C.c_uint32, C.c_uint32, _vp, C.c_uint64, C.POINTER(C.c_uint64),
         _vp, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)],
    ),
    "tsb_transpose_plan_create": (C.c_int, [C.c_int, C.POINTER(Rect), C.c_uint64, C.c_uint32, C.POINTER(C.c_uint64)]),
    "tsb_transpose_compile_host": (
        C.c_int, [C.c_int, C.POINTER(Rect), C.c_uint64, C.c_uint32, _vp, C.c_uint64, C.POINTER(C.c_uint64)],
    ),
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
# fp8 has a code only as one side of a cast: moved as itself it is an opaque byte (dtype_code -> TSB_U8)
_CAST_CODES = {**_FLOAT_CODES, torch.float8_e4m3fn: TSB_F8E4M3, torch.float8_e5m2: TSB_F8E5M2}
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


def cast_code(dtype: torch.dtype) -> int:
    """TSB_* code of `dtype` as one side of a fused cast (fp8 included)."""
    code = _CAST_CODES.get(dtype)
    if code is None:
        raise TypeError(f"no cast code for {dtype}")
    return code


def cast_supported(src: torch.dtype, dst: torch.dtype) -> bool:
    if src == dst:
        return True
    if src not in _CAST_CODES or dst not in _CAST_CODES:
        return False
    return bool(lib().tsb_cast_supported(_CAST_CODES[src], _CAST_CODES[dst]))


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


def _plan_create(fn, *args, flags: int = 0) -> int:
    """One of the tsb_*_plan_create calls of the scaled fp8 plans -> plan id."""
    out = C.c_uint64(0)
    check(fn(*args, flags, C.byref(out)))
    return int(out.value)


def _structs(struct, items: list) -> tuple:
    """``items`` as a C array of ``struct`` (at least one element) and their number."""
    return (struct * max(1, len(items)))(*items), len(items)


def _compile_host(fn, args: tuple, dtypes: list, n_groups: bool, flags: int = 0) -> list:
    """Call a tsb_*_compile_host for its record counts, then for its tables -> one numpy record array per
    table (dtypes: their layouts, in output order), then the number of two-pass groups if the call reports it."""
    import numpy as np

    counts = [C.c_uint64(0) for _ in dtypes]
    ng = C.c_uint64(0)

    def call(tables):
        outs = []
        for t, c in zip(tables, counts):
            outs += [None, 0, C.byref(c)] if t is None else [t.ctypes.data, c.value, C.byref(c)]
        check(fn(*args, flags, *outs, *([C.byref(ng)] if n_groups else [])))

    call([None] * len(dtypes))
    tables = [np.zeros(max(1, c.value), dtype=dt) for c, dt in zip(counts, dtypes)]
    call(tables)
    return [t[: c.value] for t, c in zip(tables, counts)] + ([int(ng.value)] if n_groups else [])


def make_target_array(n: int):
    return (BqTarget * n)()


def block_fp8_plan_create(device: int, rects, n: int, targets: list, flags: int = 0) -> int:
    return _plan_create(lib().tsb_block_fp8_plan_create, device, rects, n, *_structs(BqTarget, targets), flags=flags)


# record layouts of tsb_block_fp8_compile_host (include/tstore_b200.h)
BQ_BLOCK_DTYPE = [("dst", "<u8"), ("scale_inv", "<u8"), ("pitch", "<u4"), ("rows", "<u2"), ("cols", "<u2"),
                  ("piece0", "<u4"), ("n_pieces", "<u2"), ("src_dtype", "<u2")]
BQ_PIECE_DTYPE = [("src", "<u8"), ("src_stride", "<i8"), ("row0", "<u2"), ("col0", "<u2"), ("rows", "<u2"),
                  ("cols", "<u2"), ("vec", "<u4"), ("pad", "<u4")]


def block_fp8_compile_host(device: int, rects, n: int, targets, n_targets: int, flags: int = 0):
    """Host-only compilation of a block-scaled fp8 pull -> (blocks, pieces) numpy record arrays."""
    return tuple(_compile_host(lib().tsb_block_fp8_compile_host, (device, rects, n, targets, n_targets),
                               [BQ_BLOCK_DTYPE, BQ_PIECE_DTYPE], False, flags))


def make_sq_target_array(n: int):
    return (SqTarget * n)()


def scaled_fp8_plan_create(device: int, rects, n: int, targets: list, flags: int = 0) -> int:
    return _plan_create(lib().tsb_scaled_fp8_plan_create, device, rects, n, *_structs(SqTarget, targets), flags=flags)


# record layouts of tsb_scaled_fp8_compile_host (include/tstore_b200.h)
SQ_BAND_DTYPE = [("dst", "<u8"), ("scale_inv", "<u8"), ("cols", "<u4"), ("rows", "<u4"), ("piece0", "<u4"),
                 ("n_pieces", "<u4"), ("src_dtype", "<u4"), ("pad", "<u4")]
SQ_PIECE_DTYPE = [("src", "<u8"), ("src_stride", "<i8"), ("row0", "<u4"), ("col0", "<u4"), ("rows", "<u4"),
                  ("cols", "<u4"), ("vec", "<u4"), ("pad", "<u4")]
SQ_TILE_DTYPE = [("src", "<u8"), ("src_stride", "<i8"), ("dst", "<u8"), ("scale_inv", "<u8"), ("pitch", "<u4"),
                 ("rows", "<u4"), ("cols", "<u4"), ("group", "<u4"), ("src_dtype", "<u4"), ("vec", "<u4")]


def scaled_fp8_compile_host(device: int, rects, n: int, targets, n_targets: int, flags: int = 0):
    """Host-only compilation of a per-channel / per-tensor scaled fp8 pull -> (bands, pieces, tiles,
    n_groups): numpy record arrays and the number of two-pass groups."""
    return tuple(_compile_host(lib().tsb_scaled_fp8_compile_host, (device, rects, n, targets, n_targets),
                               [SQ_BAND_DTYPE, SQ_PIECE_DTYPE, SQ_TILE_DTYPE], True, flags))


def make_dq_source_array(n: int):
    return (DqSource * n)()


def dequant_fp8_plan_create(device: int, rects, n: int, sources: list, flags: int = 0) -> int:
    return _plan_create(lib().tsb_dequant_fp8_plan_create, device, rects, n, *_structs(DqSource, sources), flags=flags)


# record layout of tsb_dequant_fp8_compile_host (include/tstore_b200.h)
DQ_TILE_DTYPE = [("src", "<u8"), ("dst", "<u8"), ("scale", "<u8"), ("src_stride", "<i8"), ("dst_stride", "<i8"),
                 ("rows", "<u4"), ("cols", "<u4"), ("scale_step", "<u2"), ("dst_dtype", "u1"), ("vec", "u1"),
                 ("pad", "<u4")]


def dequant_fp8_compile_host(device: int, rects, n: int, sources, n_sources: int, flags: int = 0):
    """Host-only compilation of a dequantising pull -> its tile table as a numpy record array."""
    return _compile_host(lib().tsb_dequant_fp8_compile_host, (device, rects, n, sources, n_sources), [DQ_TILE_DTYPE],
                         False, flags)[0]


def requant_fp8_plan_create(device: int, rects, n: int, sources: list, targets: list, flags: int = 0) -> int:
    for i in range(n):  # a same-dtype fp8 window is an opaque byte move to build_rects
        rects[i].src_dtype = rects[i].dst_dtype = TSB_F8E4M3
    return _plan_create(lib().tsb_requant_fp8_plan_create, device, rects, n, *_structs(DqSource, sources),
                        *_structs(SqTarget, targets), flags=flags)


# record layouts of tsb_requant_fp8_compile_host (include/tstore_b200.h)
RQ_UNIT_DTYPE = [("dst", "<u8"), ("scale_inv", "<u8"), ("pitch", "<u4"), ("rows", "<u4"), ("cols", "<u4"),
                 ("piece0", "<u4"), ("n_pieces", "<u4"), ("per_row", "<u4")]
RQ_PIECE_DTYPE = [("src", "<u8"), ("src_stride", "<i8"), ("scale", "<u8"), ("row0", "<u4"), ("col0", "<u4"),
                  ("rows", "<u4"), ("cols", "<u4"), ("scale_step", "<u4"), ("vec", "<u4"), ("col_phase", "<u4"),
                  ("col_blocks", "<u4")]
RQ_TILE_DTYPE = [("src", "<u8"), ("src_stride", "<i8"), ("scale", "<u8"), ("dst", "<u8"), ("scale_inv", "<u8"),
                 ("pitch", "<u4"), ("rows", "<u4"), ("cols", "<u4"), ("group", "<u4"), ("scale_step", "<u4"),
                 ("vec", "<u4")]


def requant_fp8_compile_host(device: int, rects, n: int, sources, n_sources: int, targets, n_targets: int,
                             flags: int = 0):
    """Host-only compilation of a requantising pull -> (units, pieces, tiles, n_groups): numpy record arrays
    and the number of two-pass groups."""
    return tuple(_compile_host(lib().tsb_requant_fp8_compile_host, (device, rects, n, sources, n_sources, targets, n_targets),
                               [RQ_UNIT_DTYPE, RQ_PIECE_DTYPE, RQ_TILE_DTYPE], True, flags))


def make_source_quant_target_array(n: int):
    return (SourceQuantTarget * n)()


def source_quant_plan_create(device: int, targets: list, flags: int = 0, dst_dtype: int = TSB_F8E4M3) -> int:
    """``dst_dtype``: the staging format, TSB_F8E4M3 or TSB_I8 (tsb_source_quant_plan_create_as)."""
    return _plan_create(lib().tsb_source_quant_plan_create_as, device, *_structs(SourceQuantTarget, targets), dst_dtype,
                        flags=flags)


# record layout of the units of tsb_source_quant_compile_host (include/tstore_b200.h); its tiles are SQ_TILE_DTYPE
SRCQ_UNIT_DTYPE = [("src", "<u8"), ("dst", "<u8"), ("scale_inv", "<u8"), ("src_pitch", "<u4"), ("dst_pitch", "<u4"),
                   ("rows", "<u4"), ("cols", "<u4"), ("per_row", "<u4"), ("src_dtype", "<u2"), ("vec", "<u2")]


def source_quant_compile_host(device: int, targets, n: int, flags: int = 0, dst_dtype: int | None = None):
    """Host-only compilation of a source-side quantisation -> (units, tiles, n_groups): numpy record arrays and
    the number of two-pass groups.  ``dst_dtype`` (TSB_F8E4M3 or TSB_I8) goes to tsb_source_quant_compile_host_as;
    None calls tsb_source_quant_compile_host."""
    if dst_dtype is None:
        fn, args = lib().tsb_source_quant_compile_host, (device, targets, n)
    else:
        fn, args = lib().tsb_source_quant_compile_host_as, (device, targets, n, dst_dtype)
    return tuple(_compile_host(fn, args, [SRCQ_UNIT_DTYPE, SQ_TILE_DTYPE], True, flags))


def transpose_plan_create(device: int, rects, n: int, flags: int = 0) -> int:
    return _plan_create(lib().tsb_transpose_plan_create, device, rects, n, flags=flags)


# record layout of tsb_transpose_compile_host (include/tstore_b200.h)
TR_TILE_DTYPE = [("src", "<u8"), ("dst", "<u8"), ("src_stride", "<i8"), ("dst_stride", "<i8"), ("rows", "<u4"),
                 ("cols", "<u4"), ("src_dtype", "u1"), ("dst_dtype", "u1"), ("vec", "u1"), ("pad0", "u1"), ("pad1", "<u4")]


def transpose_compile_host(device: int, rects, n: int, flags: int = 0):
    """Host-only compilation of a transposing pull -> its tile table as a numpy record array."""
    return _compile_host(lib().tsb_transpose_compile_host, (device, rects, n), [TR_TILE_DTYPE], False, flags)[0]


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

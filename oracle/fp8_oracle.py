"""TEST INFRASTRUCTURE ONLY -- ctypes loader for the fp8 CPU oracle (oracle/fp8_ref.c).

fp8_ref.c compiles copy_rects_ref.c in unchanged and adds the fp8 casts (float8_e4m3fn, float8_e5m2
<-> f32, bf16, f16) with torch's .to() semantics: a flat converter, a rectangle mover and a replay
interpreter for compiled plan tables, each accepting every pair copy_rects_ref.c accepts plus fp8.
"""

from __future__ import annotations

import ctypes as C
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.path.join(HERE, "_build", "liboracle_fp8.so")

_lib = None


def build(force: bool = False) -> str:
    srcs = [os.path.join(HERE, "fp8_ref.c"), os.path.join(HERE, "copy_rects_ref.c")]
    hdr = os.path.join(os.path.dirname(HERE), "include", "tstore_b200.h")
    stale = (not os.path.exists(LIB)) or os.path.getmtime(LIB) < max(os.path.getmtime(p) for p in srcs + [hdr])
    if force or stale:
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        cmd = ["gcc", "-O2", "-fPIC", "-shared", "-pthread", "-std=gnu11", "-I", os.path.dirname(hdr), "-I", HERE,
               "-o", LIB + ".tmp", srcs[0], "-lm"]
        proc = subprocess.run(cmd, capture_output=True, text=True)
        if proc.returncode != 0:
            raise RuntimeError(f"fp8 oracle build failed:\n{proc.stdout}\n{proc.stderr}")
        os.replace(LIB + ".tmp", LIB)
    return LIB


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        build()
        h = C.CDLL(LIB)
        h.oracle_fp8_convert.restype = C.c_int
        h.oracle_fp8_convert.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_uint64, C.c_int]
        h.oracle_fp8_copy_rects.restype = C.c_int
        h.oracle_fp8_copy_rects.argtypes = [C.c_void_p, C.c_uint64, C.c_int]
        h.oracle_fp8_replay_plan.restype = C.c_int
        h.oracle_fp8_replay_plan.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_uint32, C.c_int]
        _lib = h
    return _lib


def convert(src_ptr: int, src_code: int, dst_ptr: int, dst_code: int, n: int, nan_mode: int = 0) -> None:
    st = lib().oracle_fp8_convert(C.c_void_p(src_ptr), src_code, C.c_void_p(dst_ptr), dst_code, n, nan_mode)
    if st != 0:
        raise RuntimeError(f"oracle_fp8_convert failed with {st}")


def copy_rects(rects, n: int, nan_mode: int = 0) -> None:
    """rects: ctypes array of tsb_rect_t (torchstore_b200._native.Rect) with host pointers."""
    st = lib().oracle_fp8_copy_rects(C.cast(rects, C.c_void_p), n, nan_mode)
    if st != 0:
        raise RuntimeError(f"oracle_fp8_copy_rects failed with {st}")


def replay_plan(rect_table, tiles, tile_units: int, nan_mode: int = 0) -> None:
    """Replay tables from tsb_plan_compile_host (numpy arrays) on host memory."""
    n_rects = rect_table.size // 192
    st = lib().oracle_fp8_replay_plan(C.c_void_p(rect_table.ctypes.data), n_rects, C.c_void_p(tiles.ctypes.data),
                                      tiles.shape[0], tile_units, nan_mode)
    if st != 0:
        raise RuntimeError(f"oracle_fp8_replay_plan failed with {st}")

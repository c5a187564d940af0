"""TEST INFRASTRUCTURE ONLY -- references of the dequantising pull (block-, channel- or tensor-scaled
float8_e4m3fn sources into bf16 / f16 / f32).

* ``dequantize``        numpy restatement: exact e4m3fn decoding, one np.float32 multiply per element, and
                        torch CPU's ``.to()`` for the final narrowing;
* ``torch_dequantize``  the torch rendering ``(q.float() * s_expanded).to(dst)`` (DeepSeek's weight_dequant)
                        on any device: the recorder of tests/golden/dequant_fp8_vectors.npz on the CPU and the
                        reference of the H100 tests;
* ``replay``            an interpreter of the tables ``tsb_dequant_fp8_compile_host`` returns, on host memory.

The formula, for element (i, j) of a source shard at global offset (r0, c0) in its last two dims (leading
dims are independent matrices; scales are anchored at the global origin and hold exactly the groups the
shard touches):
    g(i, j) = block:   ((r0 + i) // 128 - r0 // 128, (c0 + j) // 128 - c0 // 128)
              channel: (i, 0)
              tensor:  ()
    y = to_dst(f32(q[b, i, j]) * scale[b, g(i, j)])
"""

from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from oracle.block_fp8_oracle import digest, synth_f32  # noqa: F401  (re-exported for the tests)

BLOCK = 128
E4M3 = torch.float8_e4m3fn
GRANULARITIES = ("block", "channel", "tensor")
DST = {"bfloat16": torch.bfloat16, "float16": torch.float16, "float32": torch.float32}


def scale_shape(granularity: str, shape, r0: int = 0, c0: int = 0) -> tuple:
    """Shape of the scale of a ``shape`` shard at global offset (r0, c0) (per tensor: ``lead``)."""
    *lead, n, k = shape
    if granularity == "block":
        return (*lead, -(-(r0 + n) // BLOCK) - r0 // BLOCK, -(-(c0 + k) // BLOCK) - c0 // BLOCK)
    if granularity == "channel":
        return (*lead, n, 1)
    if granularity == "tensor":
        return tuple(lead)
    raise ValueError(f"granularity must be one of {GRANULARITIES}, not {granularity!r}")


def decode_e4m3(q: np.ndarray) -> np.ndarray:
    """e4m3fn bytes -> exact float32 values (0x7F / 0xFF are NaN; no Inf)."""
    b = np.asarray(q, dtype=np.uint8).astype(np.int64)
    sign = np.where(b & 0x80, -1.0, 1.0)
    e, m = (b >> 3) & 0xF, b & 7
    mag = np.where(e == 0, m / 8.0 * 2.0 ** -6, (1.0 + m / 8.0) * np.exp2(e - 7.0))
    out = (sign * mag).astype(np.float32)
    out[(e == 15) & (m == 7)] = np.nan
    return out


def expand(scale: np.ndarray, shape, granularity: str, r0: int = 0, c0: int = 0) -> np.ndarray:
    """The scale of every element of a ``shape`` shard (float32, broadcast to ``shape``)."""
    *lead, n, k = shape
    s = np.asarray(scale, dtype=np.float32).reshape(scale_shape(granularity, shape, r0, c0))
    if granularity == "block":
        gr = (r0 + np.arange(n)) // BLOCK - r0 // BLOCK
        gc = (c0 + np.arange(k)) // BLOCK - c0 // BLOCK
        return s[..., gr[:, None], gc[None, :]]
    if granularity == "channel":
        return np.broadcast_to(s, shape)
    return np.broadcast_to(s.reshape(tuple(lead) + (1, 1)), shape)


def narrow(y: np.ndarray, dst: str) -> np.ndarray:
    """float32 values -> raw bits of ``dst`` (uint16 for bf16/f16, uint32 for f32) with torch CPU's .to()."""
    if dst == "float32":
        return np.ascontiguousarray(y, dtype=np.float32).view(np.uint32)
    t = torch.from_numpy(np.ascontiguousarray(y, dtype=np.float32)).to(DST[dst])
    return t.view(torch.int16).numpy().view(np.uint16)


def dequantize(q: np.ndarray, scale: np.ndarray, granularity: str, r0: int = 0, c0: int = 0,
               dst: str = "bfloat16") -> np.ndarray:
    """q: e4m3fn bytes [..., N, K] -> raw bits of the dequantised ``dst`` values."""
    x = decode_e4m3(q)
    with np.errstate(all="ignore"):
        y = (x * expand(scale, x.shape, granularity, r0, c0)).astype(np.float32)
    return narrow(y, dst)


def torch_dequantize(q: torch.Tensor, scale: torch.Tensor, granularity: str, r0: int = 0, c0: int = 0,
                     dst: torch.dtype = torch.bfloat16) -> torch.Tensor:
    """``(q.float() * s_expanded).to(dst)`` on q's device."""
    *lead, n, k = q.shape
    s = scale.float().reshape(scale_shape(granularity, tuple(q.shape), r0, c0))
    if granularity == "block":
        gr = torch.div(r0 + torch.arange(n, device=q.device), BLOCK, rounding_mode="floor") - r0 // BLOCK
        gc = torch.div(c0 + torch.arange(k, device=q.device), BLOCK, rounding_mode="floor") - c0 // BLOCK
        s = s[..., gr[:, None], gc[None, :]]
    elif granularity == "tensor":
        s = s.reshape(*lead, 1, 1)
    return (q.float() * s).to(dst)


def fp8_of(shape, seed: int) -> torch.Tensor:
    """Deterministic finite e4m3fn values (|x| <= 256) rebuilt from an integer hash."""
    return synth_f32(shape, seed).to(E4M3)


def scale_of(shape, seed: int) -> torch.Tensor:
    """Deterministic positive float32 scales around amax/448 of typical weights."""
    return synth_f32(shape, seed, spread=4).abs() * np.float32(0.02 / 448) + np.float32(1e-7)


# the scale set of the all-bytes table: every e4m3fn byte times each of these
SCALE_SET = np.array([1.0, 2.0 ** -7, 2.0 ** 9, 0.0123 / 448, 2.0 ** -140, 2.0 ** -120, 1000.0, 7.589e35, 0.0, -0.5,
                      np.inf, np.nan], dtype=np.float32)


def fixture_inputs() -> list[tuple[str, str, int, int, torch.Tensor, torch.Tensor]]:
    """(name, granularity, r0, c0, q, scale) of tests/golden/dequant_fp8_vectors.npz: all 256 e4m3fn bytes per
    channel against SCALE_SET (f32-subnormal products at 2^-140 and 2^-120, f16 overflow at 1000, bf16 overflow
    at 7.589e35, 0, a negative scale, Inf and NaN); each granularity on a matrix at an unaligned (r0, c0); and
    MoE [E, N, K] stacks."""
    q = torch.arange(256, dtype=torch.uint8).repeat(len(SCALE_SET), 1).view(E4M3)
    out = [("all_bytes", "channel", 0, 0, q, torch.from_numpy(SCALE_SET.copy()).reshape(-1, 1))]
    for k, g in enumerate(GRANULARITIES):
        for name, shape, r0, c0 in (("matrix", (300, 260), 37, 70), ("aligned", (256, 384), 0, 0),
                                    ("moe", (3, 130, 260), 100, 5)):
            seed = 5000 + 100 * k + 10 * len(out)
            out.append((f"{name}_{g}", g, r0, c0, fp8_of(shape, seed), scale_of(scale_shape(g, shape, r0, c0), seed + 1)))
    return out


_DST = {4: ("float16", 2), 5: ("bfloat16", 2), 6: ("float32", 4)}  # TSB_F16, TSB_BF16, TSB_F32


def _host(ptr: int, nbytes: int) -> np.ndarray:
    return np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(ptr))


def replay(tiles: np.ndarray) -> None:
    """Execute compiled dequant tiles on host memory: every row of a tile reads its fp8 bytes, multiplies
    them by the scale at ``scale + r * scale_step`` and stores the narrowed values."""
    for t in tiles:
        dst, es = _DST[int(t["dst_dtype"])]
        rows, cols = int(t["rows"]), int(t["cols"])
        for r in range(rows):
            q = _host(int(t["src"]) + r * int(t["src_stride"]), cols)
            s = _host(int(t["scale"]) + r * int(t["scale_step"]), 4).view(np.float32)[0]
            with np.errstate(all="ignore"):
                y = (decode_e4m3(q) * s).astype(np.float32)
            _host(int(t["dst"]) + r * int(t["dst_stride"]), cols * es)[:] = narrow(y, dst).view(np.uint8)

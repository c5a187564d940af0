"""TEST INFRASTRUCTURE ONLY -- references of the requantising pull (block-, channel- or tensor-scaled
float8_e4m3fn sources into block-, channel- or tensor-scaled float8_e4m3fn destinations).

* ``requantize``        numpy composition: ``dequant_fp8_oracle.dequantize(..., dst="float32")`` followed by
                        ``block_fp8_oracle.quantize`` / ``scaled_fp8_oracle.quantize``;
* ``torch_requantize``  the torch rendering: ``torch_dequantize(..., torch.float32)`` followed by the
                        quantisers' ``torch_quantize``, on any device: the recorder of
                        tests/golden/requant_fp8_vectors.npz on the CPU and the reference of the H100 tests;
* ``replay``            an interpreter of the tables ``tsb_requant_fp8_compile_host`` returns, on host memory.

The formula: every element of the destination window is x = f32(q) * s_src (the value a dequantising pull
into f32 writes, with the scale of the shard the byte is read from), and the window is quantised with the
destination's granularity as if x were an f32 source:
    amax = max |x| over the group (NaN if any x is NaN); amax_c = max(amax, float32(1e-4))
    q' = e4m3fn(rn(x * (448 / amax_c))); scale_inv = amax_c / 448
"""

from __future__ import annotations

import ctypes as C
from collections import defaultdict

import numpy as np
import torch

from oracle import block_fp8_oracle, scaled_fp8_oracle
from oracle.block_fp8_oracle import digest  # noqa: F401  (re-exported for the tests)
from oracle.dequant_fp8_oracle import (GRANULARITIES, decode_e4m3, dequantize, fp8_of, scale_of, scale_shape,
                                       torch_dequantize)

E4M3 = torch.float8_e4m3fn
PAIRS = tuple((s, d) for s in GRANULARITIES for d in GRANULARITIES)  # (source, destination) granularities


def canonical_nan(q: np.ndarray) -> np.ndarray:
    """e4m3fn bytes with every NaN (0x7F / 0xFF) written as 0x7F."""
    q = np.array(q, dtype=np.uint8)
    q[(q & 0x7F) == 0x7F] = 0x7F
    return q


def quantize(x: np.ndarray, granularity: str) -> tuple[np.ndarray, np.ndarray]:
    """float32 x [..., N, K] -> (q uint8, scale_inv float32) with the destination's formula."""
    if granularity == "block":
        return block_fp8_oracle.quantize(x)
    return scaled_fp8_oracle.quantize(x, granularity)


def requantize(q: np.ndarray, scale: np.ndarray, src_g: str, r0: int, c0: int, dst_g: str) -> tuple[np.ndarray, np.ndarray]:
    """q: e4m3fn bytes [..., N, K] of a window at global offset (r0, c0) with its source scale -> (q', scale_inv)
    of a ``dst_g`` destination holding exactly that window."""
    x = dequantize(q, scale, src_g, r0, c0, "float32").view(np.float32)
    return quantize(x, dst_g)


def torch_requantize(q: torch.Tensor, scale: torch.Tensor, src_g: str, r0: int, c0: int,
                     dst_g: str) -> tuple[torch.Tensor, torch.Tensor]:
    """The two-step torch rendering on q's device -> (q' float8_e4m3fn, scale_inv float32)."""
    x = torch_dequantize(q, scale, src_g, r0, c0, torch.float32)
    if dst_g == "block":
        return block_fp8_oracle.torch_quantize(x)
    return scaled_fp8_oracle.torch_quantize(x, dst_g)


# source scales with a non-finite entry: poisons the groups it reaches
SCALE_POISON = np.array([np.inf, np.nan], dtype=np.float32)


def fixture_inputs() -> list[tuple[str, str, str, int, int, torch.Tensor, torch.Tensor]]:
    """(name, source granularity, destination granularity, r0, c0, q, scale) of
    tests/golden/requant_fp8_vectors.npz: every (source, destination) pair on a [300, 260] window at the
    unaligned global offset (37, 70), on a [3, 130, 260] MoE stack at (100, 5), and one block-scaled window
    whose scale holds Inf and NaN, into each destination granularity."""
    out = []
    for k, (sg, dg) in enumerate(PAIRS):
        for name, shape, r0, c0 in (("matrix", (300, 260), 37, 70), ("moe", (3, 130, 260), 100, 5)):
            seed = 7000 + 100 * k + 10 * len(out)
            out.append((f"{name}_{sg}_{dg}", sg, dg, r0, c0, fp8_of(shape, seed), scale_of(scale_shape(sg, shape, r0, c0), seed + 1)))
    for dg in GRANULARITIES:
        shape = (300, 260)
        s = scale_of(scale_shape("block", shape, 37, 70), 7901)
        s[1, 0], s[2, 2] = float(SCALE_POISON[0]), float(SCALE_POISON[1])
        out.append((f"poison_block_{dg}", "block", dg, 37, 70, fp8_of(shape, 7900), s))
    return out


def _host(ptr: int, nbytes: int) -> np.ndarray:
    return np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(ptr))


def _x(src: int, stride: int, scale: int, step: int, rows: int, cols: int, col_phase: int = 0,
       col_blocks: int = 0) -> np.ndarray:
    """The scaled values of a source rectangle: element (r, c) under the float32 scale at
    scale + r * step (+ 4 * ((col_phase + c) // 128) with col_blocks)."""
    x = np.zeros((rows, cols), dtype=np.float32)
    groups = (col_phase + np.arange(cols)) // 128 if col_blocks else np.zeros(cols, dtype=np.int64)
    for r in range(rows):
        s = _host(scale + r * step, 4 * (int(groups[-1]) + 1)).view(np.float32)[groups]
        with np.errstate(all="ignore"):
            x[r] = decode_e4m3(_host(src + r * stride, cols)) * s
    return x


def replay(units: np.ndarray, pieces: np.ndarray, tiles: np.ndarray, n_groups: int) -> None:
    """Execute compiled requant tables on host memory.  Units: gather the pieces' scaled values, quantise the
    block (one group) or every row (per_row), store the bytes and the scale_inv.  Tiles: pass 1 folds each
    group's amax, pass 2 quantises every tile with its group's scale; the tile holding a non-zero scale_inv
    address stores it."""
    for u in units:
        rows, cols, pitch = int(u["rows"]), int(u["cols"]), int(u["pitch"])
        x = np.full((rows, cols), np.nan, dtype=np.float32)
        for p in pieces[int(u["piece0"]): int(u["piece0"]) + int(u["n_pieces"])]:
            r0, c0, pr, pc = (int(p[f]) for f in ("row0", "col0", "rows", "cols"))
            x[r0: r0 + pr, c0: c0 + pc] = _x(int(p["src"]), int(p["src_stride"]), int(p["scale"]), int(p["scale_step"]), pr, pc,
                                             int(p["col_phase"]), int(p["col_blocks"]))
        q, s = scaled_fp8_oracle.quantize(x, "channel" if int(u["per_row"]) else "tensor")
        for r in range(rows):
            _host(int(u["dst"]) + r * pitch, cols)[:] = q[r]
        _host(int(u["scale_inv"]), s.size * 4)[:] = np.ascontiguousarray(s, dtype=np.float32).reshape(-1).view(np.uint8)
    values = [_x(int(t["src"]), int(t["src_stride"]), int(t["scale"]), int(t["scale_step"]), int(t["rows"]), int(t["cols"]))
              for t in tiles]
    amax = defaultdict(lambda: np.float32(0))
    for t, x in zip(tiles, values):
        g = int(t["group"])
        assert g < n_groups
        amax[g] = np.maximum(amax[g], np.abs(x).max())  # NaN propagates
    for t, x in zip(tiles, values):
        scale, scale_inv = scaled_fp8_oracle.scales_of_amax(amax[int(t["group"])])
        with np.errstate(all="ignore"):
            q = scaled_fp8_oracle.narrow((x * scale).astype(np.float32))
        for r in range(int(t["rows"])):
            _host(int(t["dst"]) + r * int(t["pitch"]), int(t["cols"]))[:] = q[r]
        if int(t["scale_inv"]):
            _host(int(t["scale_inv"]), 4)[:] = np.asarray(scale_inv, dtype=np.float32).reshape(1).view(np.uint8)

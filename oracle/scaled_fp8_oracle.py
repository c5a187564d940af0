"""TEST INFRASTRUCTURE ONLY -- per-channel and per-tensor scaled FP8 (float32 scale_inv per row / per
matrix) references.

* ``quantize``        numpy float32 restatement of the formula (true IEEE divisions), with torch CPU's
                      ``.to(float8_e4m3fn)`` (the fp8 golden reference) for the final narrowing;
* ``torch_quantize``  the same formula in torch tensor/tensor ops, on any device: the recorder of
                      tests/golden/scaled_fp8_vectors.npz on the CPU and the reference of the H100 tests;
* ``replay``          an interpreter of the tables ``tsb_scaled_fp8_compile_host`` returns, on host memory.

The formula is block_fp8_oracle's over another group -- one row of the last two dims ("channel") or the
whole [rows, cols] matrix ("tensor"); leading dims are independent matrices:
    amax = max |x| (NaN if any x is NaN); amax_c = max(amax, float32(1e-4)) (NaN stays NaN)
    scale = 448 / amax_c; q = e4m3fn(rn(x * scale)); scale_inv = amax_c / 448
scale_inv has shape lead + (N, 1) per channel and lead per tensor.
"""

from __future__ import annotations

import ctypes as C
from collections import defaultdict

import numpy as np
import torch

from oracle.block_fp8_oracle import bits_of, digest, synth_f32, widen  # noqa: F401  (re-exported for the tests)

E4M3 = torch.float8_e4m3fn
GRANULARITIES = ("channel", "tensor")
_CLAMP = np.float32(1e-4)
_FMAX = np.float32(448.0)


def _dims(granularity: str) -> tuple:
    if granularity not in GRANULARITIES:
        raise ValueError(f"granularity must be one of {GRANULARITIES}, not {granularity!r}")
    return (-1,) if granularity == "channel" else (-2, -1)


def scales_of_amax(amax: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """float32 amax -> (scale, scale_inv), both correctly rounded f32 divisions; NaN stays NaN."""
    with np.errstate(all="ignore"):
        amax_c = np.maximum(np.asarray(amax, dtype=np.float32), _CLAMP)  # NaN propagates
        return (_FMAX / amax_c).astype(np.float32), (amax_c / _FMAX).astype(np.float32)


def narrow(prod: np.ndarray) -> np.ndarray:
    """float32 products -> e4m3fn bytes with torch CPU's .to() rounding."""
    return torch.from_numpy(np.ascontiguousarray(prod, dtype=np.float32)).to(E4M3).view(torch.uint8).numpy()


def quantize(x: np.ndarray, granularity: str) -> tuple[np.ndarray, np.ndarray]:
    """x: float32 array [..., N, K] (the exactly widened source values) -> (q as uint8, scale_inv float32)."""
    x = np.asarray(x, dtype=np.float32)
    amax = np.abs(x).max(axis=_dims(granularity), keepdims=True)  # NaN propagates
    scale, scale_inv = scales_of_amax(amax)
    with np.errstate(all="ignore"):
        q = narrow((x * scale).astype(np.float32))
    return q, scale_inv if granularity == "channel" else scale_inv.reshape(x.shape[:-2])


def torch_quantize(x: torch.Tensor, granularity: str) -> tuple[torch.Tensor, torch.Tensor]:
    """The formula in torch tensor/tensor ops on x's device -> (q float8_e4m3fn, scale_inv float32).
    ``448.0 / amax`` would be reciprocal-then-multiply (two roundings): hence full_like(448).div."""
    xf = x.float()
    amax = xf.abs().amax(dim=_dims(granularity), keepdim=True)
    amax_c = torch.maximum(amax, torch.full_like(amax, 1e-4))
    fmax = torch.full_like(amax_c, 448.0)
    scale_inv = amax_c.div(fmax)
    q = xf.mul(fmax.div(amax_c)).to(E4M3)
    return q, scale_inv if granularity == "channel" else scale_inv.reshape(xf.shape[:-2])


def fixture_inputs() -> list[tuple[str, torch.Tensor]]:
    """The source tensors of tests/golden/scaled_fp8_vectors.npz, each recorded per channel and per tensor:
    random, ragged, single-row and 3-D [3, 130, 260] bf16/f16/f32 tensors; all-zero rows and an all-zero
    matrix (the 1e-4 clamp), +-0 and subnormal rows; bf16 values near 3e38; rows longer than the row-staged
    kernel's 32 KiB stage (the two-pass path per channel); a row with +-Inf and a row with a NaN."""
    out = []
    for k, dtype in enumerate((torch.bfloat16, torch.float16, torch.float32)):
        name = str(dtype).replace("torch.", "")
        seed = 100 * k + 1000
        out.append((f"random_{name}_128x384", synth_f32((128, 384), seed + 1).to(dtype)))
        out.append((f"ragged_{name}_300x200", synth_f32((300, 200), seed + 2).to(dtype)))
        out.append((f"ragged_{name}_129x257", synth_f32((129, 257), seed + 3).to(dtype)))
        out.append((f"row_{name}_1x16", synth_f32((1, 16), seed + 4).to(dtype)))
        out.append((f"moe_{name}_3x130x260", synth_f32((3, 130, 260), seed + 5).to(dtype)))
        # rows 0..7 zero, 8..15 +-0 only, 16..63 subnormal-sized, 64.. tiny values
        x = synth_f32((128, 96), seed + 6)
        x[:8] = 0
        x[8:16] = torch.where(synth_f32((8, 96), seed + 7) < 0, -0.0, 0.0)
        x[16:64] = synth_f32((48, 96), seed + 8, spread=0) * torch.finfo(dtype).tiny
        x[64:] = synth_f32((64, 96), seed + 9, spread=0) * 1e-6
        out.append((f"zeros_subnormals_{name}", x.to(dtype)))
        out.append((f"zero_matrix_{name}", torch.zeros(4, 64, dtype=dtype)))
        long_cols = 16400 if dtype != torch.float32 else 8200  # 32800 source bytes per row
        out.append((f"long_rows_{name}_3x{long_cols}", synth_f32((3, long_cols), seed + 10).to(dtype)))
    # bf16 values near 3e38 (the top of bf16's range; 448 / amax stays a normal f32)
    x = (synth_f32((200, 300), 1301, spread=0).abs() * 0.4e38 + 2.9e38).to(torch.bfloat16)
    x[::3] = -x[::3]
    out.append(("huge_bfloat16", x))
    # non-finite rows: +-Inf in row 5, a NaN in row 100, finite rows beside them
    for k, dtype in enumerate((torch.bfloat16, torch.float32)):
        x = synth_f32((130, 130), 1400 + k).to(dtype)
        x[5, 7] = float("inf")
        x[5, 100] = float("-inf")
        x[100, 3] = float("nan")
        out.append((f"nonfinite_{str(dtype).replace('torch.', '')}", x))
    return out


_SRC = {4: ("float16", 2), 5: ("bfloat16", 2), 6: ("float32", 4)}  # TSB_F16, TSB_BF16, TSB_F32


def _host(ptr: int, nbytes: int) -> np.ndarray:
    return np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(ptr))


def _gather(src: int, stride: int, rows: int, cols: int, es: int) -> np.ndarray:
    bits = np.zeros((rows, cols), dtype=np.uint16 if es == 2 else np.uint32)
    for r in range(rows):
        bits[r] = _host(src + r * stride, cols * es).view(bits.dtype)
    return bits


def replay(bands: np.ndarray, pieces: np.ndarray, tiles: np.ndarray, n_groups: int) -> None:
    """Execute compiled band/piece/tile tables on host memory.  Bands: gather the pieces, quantise
    every row with its own scale, store the rows and one scale_inv per row.  Tiles: pass 1 folds each
    group's amax over its tiles, pass 2 quantises every tile with its group's scale and the tile holding
    a non-zero scale_inv address stores the group's scale_inv."""
    for b in bands:
        dtype, es = _SRC[int(b["src_dtype"])]
        rows, cols = int(b["rows"]), int(b["cols"])
        bits = np.zeros((rows, cols), dtype=np.uint16 if es == 2 else np.uint32)
        for p in pieces[int(b["piece0"]): int(b["piece0"]) + int(b["n_pieces"])]:
            r0, c0, pr, pc = (int(p[f]) for f in ("row0", "col0", "rows", "cols"))
            bits[r0: r0 + pr, c0: c0 + pc] = _gather(int(p["src"]), int(p["src_stride"]), pr, pc, es)
        q, s = quantize(widen(bits, dtype), "channel")
        for r in range(rows):
            _host(int(b["dst"]) + r * cols, cols)[:] = q[r]
        _host(int(b["scale_inv"]), 4 * rows)[:] = s.reshape(-1).view(np.uint8)
    values = [widen(_gather(int(t["src"]), int(t["src_stride"]), int(t["rows"]), int(t["cols"]), _SRC[int(t["src_dtype"])][1]),
                    _SRC[int(t["src_dtype"])][0]) for t in tiles]
    amax = defaultdict(lambda: np.float32(0))
    for t, x in zip(tiles, values):
        g = int(t["group"])
        assert g < n_groups
        amax[g] = np.maximum(amax[g], np.abs(x).max())  # NaN propagates
    for t, x in zip(tiles, values):
        scale, scale_inv = scales_of_amax(amax[int(t["group"])])
        with np.errstate(all="ignore"):
            q = narrow((x * scale).astype(np.float32))
        for r in range(int(t["rows"])):
            _host(int(t["dst"]) + r * int(t["pitch"]), int(t["cols"]))[:] = q[r]
        if int(t["scale_inv"]):
            _host(int(t["scale_inv"]), 4)[:] = np.asarray(scale_inv, dtype=np.float32).reshape(1).view(np.uint8)

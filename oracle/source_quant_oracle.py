"""TEST INFRASTRUCTURE ONLY -- source-side quantisation references: a bf16/f16/f32 shard at global offset
(row0, col0) of its last two dims, quantised into block-, channel- or tensor-scaled float8_e4m3fn with
shard-local groups anchored at the global origin.

* ``quantize``        numpy restatement: the per-group formula of block_fp8_oracle / scaled_fp8_oracle over
                      the shard-local groups;
* ``torch_quantize``  the same in torch tensor/tensor ops, on any device: the recorder of
                      tests/golden/source_quant_vectors.npz on the CPU and the reference of the H100 tests;
* ``replay``          an interpreter of the tables ``tsb_source_quant_compile_host`` returns, on host memory.

Groups: per block, the part of a global 128x128 block inside the shard (scale shape
lead + (ceil((row0+N)/128) - row0//128, ceil((col0+K)/128) - col0//128)); per channel, the shard's part of one
row (lead + (N, 1)); per tensor, the shard's [N, K] matrix (lead).  The shard's block groups are the blocks
of the shard placed at (row0 % 128, col0 % 128) of a zero-padded frame: padding with zeros changes no
group's max |x|.
"""

from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from oracle import block_fp8_oracle, scaled_fp8_oracle
from oracle.block_fp8_oracle import BLOCK, bits_of, digest, synth_f32, widen  # noqa: F401  (re-exported for the tests)

GRANULARITIES = ("block", "channel", "tensor")


def quantize(x: np.ndarray, granularity: str, row0: int = 0, col0: int = 0) -> tuple[np.ndarray, np.ndarray]:
    """x: float32 [..., N, K] (the exactly widened shard) -> (q as uint8, scale_inv float32)."""
    x = np.asarray(x, dtype=np.float32)
    if granularity != "block":
        return scaled_fp8_oracle.quantize(x, granularity)
    *lead, n, k = x.shape
    ph, pw = row0 % BLOCK, col0 % BLOCK
    frame = np.zeros(tuple(lead) + (ph + n, pw + k), dtype=np.float32)
    frame[..., ph:, pw:] = x
    q, s = block_fp8_oracle.quantize(frame)
    return np.ascontiguousarray(q[..., ph:, pw:]), s


def torch_quantize(x: torch.Tensor, granularity: str, row0: int = 0, col0: int = 0) -> tuple[torch.Tensor, torch.Tensor]:
    """The formula in torch tensor/tensor ops on x's device -> (q float8_e4m3fn, scale_inv float32)."""
    if granularity != "block":
        return scaled_fp8_oracle.torch_quantize(x, granularity)
    ph, pw = row0 % BLOCK, col0 % BLOCK
    frame = torch.nn.functional.pad(x.float(), (pw, 0, ph, 0))
    q, s = block_fp8_oracle.torch_quantize(frame)
    return q[..., ph:, pw:].contiguous(), s


def fixture_inputs() -> list[tuple[str, torch.Tensor, str, int, int]]:
    """The cases of tests/golden/source_quant_vectors.npz as (name, shard, granularity, row0, col0): every
    granularity x {bf16, f16, f32} at shard offsets (0, 0), (37, 70) and (128, 256); a [3, 130, 260] stack at
    (100, 5); a shard with +-Inf and NaN groups, an all-zero group and subnormal magnitudes."""
    out = []
    for k, dtype in enumerate((torch.bfloat16, torch.float16, torch.float32)):
        name = str(dtype).replace("torch.", "")
        for gi, g in enumerate(GRANULARITIES):
            seed = 2000 + 100 * k + 10 * gi
            for j, (r0, c0) in enumerate(((0, 0), (37, 70), (128, 256))):
                out.append((f"{g}_{name}_300x200_at_{r0}_{c0}", synth_f32((300, 200), seed + j).to(dtype), g, r0, c0))
            out.append((f"{g}_{name}_moe_3x130x260_at_100_5", synth_f32((3, 130, 260), seed + 5).to(dtype), g, 100, 5))
            # at (37, 70): rows 0..91 lie in the first block row.  Block (0, 0) of the shard (rows 0..91,
            # cols 0..58) is all zero, rows 91..100 hold subnormal magnitudes, rows 100..110 tiny values,
            # row 150 has +-Inf, row 200 a NaN
            x = synth_f32((256, 200), seed + 6)
            x[:91, :58] = 0
            x[91:100] = synth_f32((9, 200), seed + 7, spread=0) * torch.finfo(dtype).tiny
            x[100:110] = synth_f32((10, 200), seed + 8, spread=0) * 1e-6
            x[150, 3] = float("inf")
            x[150, 190] = float("-inf")
            x[200, 77] = float("nan")
            out.append((f"{g}_{name}_special_at_37_70", x.to(dtype), g, 37, 70))
    return out


_SRC = {4: ("float16", 2), 5: ("bfloat16", 2), 6: ("float32", 4)}  # TSB_F16, TSB_BF16, TSB_F32


def _host(ptr: int, nbytes: int) -> np.ndarray:
    return np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(ptr))


def replay(units: np.ndarray, tiles: np.ndarray, n_groups: int) -> None:
    """Execute compiled unit/tile tables on host memory.  Units: read the rows, quantise them as one group
    (a block) or one group per row (a band), store the fp8 rows and the scale_inv(s).  Tiles: the two-pass
    path, interpreted by scaled_fp8_oracle.replay."""
    for u in units:
        dtype, es = _SRC[int(u["src_dtype"])]
        rows, cols = int(u["rows"]), int(u["cols"])
        bits = np.zeros((rows, cols), dtype=np.uint16 if es == 2 else np.uint32)
        for r in range(rows):
            bits[r] = _host(int(u["src"]) + r * int(u["src_pitch"]), cols * es).view(bits.dtype)
        q, s = scaled_fp8_oracle.quantize(widen(bits, dtype), "channel" if int(u["per_row"]) else "tensor")
        for r in range(rows):
            _host(int(u["dst"]) + r * int(u["dst_pitch"]), cols)[:] = q[r]
        s = np.asarray(s, dtype=np.float32).reshape(-1)
        _host(int(u["scale_inv"]), 4 * s.size)[:] = s.view(np.uint8)
    scaled_fp8_oracle.replay((), (), tiles, n_groups)


def element_scales(s: np.ndarray, granularity: str, shape: tuple, row0: int = 0, col0: int = 0) -> np.ndarray:
    """The scale_inv of every element of a ``shape`` shard at (row0, col0): ``s`` expanded over its groups."""
    s = np.asarray(s)
    *lead, n, k = shape
    if granularity == "tensor":
        return np.broadcast_to(s.reshape(tuple(lead) + (1, 1)), tuple(shape))
    if granularity == "channel":
        return np.broadcast_to(s.reshape(tuple(lead) + (n, 1)), tuple(shape))
    rows = (row0 + np.arange(n)) // BLOCK - row0 // BLOCK
    cols = (col0 + np.arange(k)) // BLOCK - col0 // BLOCK
    return s[..., rows[:, None], cols[None, :]]

"""TEST INFRASTRUCTURE ONLY -- block-scaled FP8 (128x128 blocks, float32 scale_inv) references.

* ``quantize``        numpy float32 restatement of the formula (true IEEE divisions), with torch CPU's
                      ``.to(float8_e4m3fn)`` (the fp8 golden reference) for the final narrowing;
* ``torch_quantize``  the same formula in torch tensor/tensor ops, on any device: the recorder of
                      tests/golden/block_fp8_vectors.npz on the CPU and the reference of the H100 tests;
* ``replay``          an interpreter of the tables ``tsb_block_fp8_compile_host`` returns, on host memory.

The formula, per 128x128 block (anchored at (0, 0) of the last two dims; edge blocks partial):
    amax = max |x| (NaN if any x is NaN); amax_c = max(amax, float32(1e-4)) (NaN stays NaN)
    scale = 448 / amax_c; q = e4m3fn(rn(x * scale)); scale_inv = amax_c / 448
Written ``448.0 / amax`` in torch is NOT this: a Python scalar over a tensor is ``reciprocal() * 448``,
two roundings.  Hence the tensor/tensor divisions below.
"""

from __future__ import annotations

import ctypes as C
import hashlib

import numpy as np
import torch

BLOCK = 128
E4M3 = torch.float8_e4m3fn
_CLAMP = np.float32(1e-4)
_FMAX = np.float32(448.0)


def _blocks(shape) -> tuple:
    *lead, n, k = shape
    return tuple(lead), -(-n // BLOCK), -(-k // BLOCK)


def _expand(s: np.ndarray, n: int, k: int) -> np.ndarray:
    return np.repeat(np.repeat(s, BLOCK, axis=-2), BLOCK, axis=-1)[..., :n, :k]


def quantize(x: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """x: float32 array [..., N, K] (the exactly widened source values) -> (q as uint8, scale_inv float32)."""
    x = np.asarray(x, dtype=np.float32)
    *lead, n, k = x.shape
    _, nb, kb = _blocks(x.shape)
    pad = np.zeros(tuple(lead) + (nb * BLOCK, kb * BLOCK), dtype=np.float32)
    pad[..., :n, :k] = np.abs(x)
    amax = pad.reshape(tuple(lead) + (nb, BLOCK, kb, BLOCK)).max(axis=(-3, -1))  # NaN propagates
    with np.errstate(all="ignore"):
        amax_c = np.maximum(amax, _CLAMP)  # NaN propagates
        scale = (_FMAX / amax_c).astype(np.float32)
        scale_inv = (amax_c / _FMAX).astype(np.float32)
        prod = (x * _expand(scale, n, k)).astype(np.float32)
    q = torch.from_numpy(np.ascontiguousarray(prod)).to(E4M3).view(torch.uint8).numpy()
    return q, scale_inv


def torch_quantize(x: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """The formula in torch tensor/tensor ops on x's device -> (q float8_e4m3fn, scale_inv float32)."""
    xf = x.float()
    *lead, n, k = xf.shape
    _, nb, kb = _blocks(xf.shape)
    pad = torch.nn.functional.pad(xf.abs(), (0, kb * BLOCK - k, 0, nb * BLOCK - n))
    amax = pad.reshape(*lead, nb, BLOCK, kb, BLOCK).amax(dim=(-3, -1))
    amax_c = torch.maximum(amax, torch.full_like(amax, 1e-4))
    fmax = torch.full_like(amax_c, 448.0)
    scale = fmax.div(amax_c)
    scale_inv = amax_c.div(fmax)
    full = scale.repeat_interleave(BLOCK, -2).repeat_interleave(BLOCK, -1)[..., :n, :k]
    return xf.mul(full).to(E4M3), scale_inv


def synth_f32(shape, seed: int, spread: int = 8) -> torch.Tensor:
    """Deterministic pseudo-random float32 values: splitmix64 of (element index, seed), no RNG state,
    so every platform and torch version rebuilds the same inputs.  Values are (2u - 1) * 2^e with u
    in (0, 1) and e uniform in [-spread, spread)."""
    n = int(np.prod(shape))
    z = np.arange(n, dtype=np.uint64) + np.uint64(seed * 0x9E3779B97F4A7C15 % 2**64)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    z = z ^ (z >> np.uint64(31))
    u = ((z >> np.uint64(11)).astype(np.float64) + 0.5) / 2.0**53
    x = 2.0 * u - 1.0
    if spread:
        x = x * np.exp2((z & np.uint64(0xFF)).astype(np.int64) % (2 * spread) - spread)
    return torch.from_numpy(x.astype(np.float32).reshape(shape))


def fixture_inputs() -> list[tuple[str, torch.Tensor]]:
    """The source tensors of tests/golden/block_fp8_vectors.npz: random bf16/f16/f32 blocks, all-zero
    blocks (the 1e-4 clamp), +-0, subnormals, bf16 values near 3e38, one +-Inf block and one NaN block,
    ragged shapes and 3-D [3, 130, 260] stacks."""
    out = []
    for k, dtype in enumerate((torch.bfloat16, torch.float16, torch.float32)):
        name = str(dtype).replace("torch.", "")
        seed = 100 * k
        out.append((f"random_{name}_128x384", synth_f32((128, 384), seed + 1).to(dtype)))
        out.append((f"ragged_{name}_300x200", synth_f32((300, 200), seed + 2).to(dtype)))
        out.append((f"ragged_{name}_129x257", synth_f32((129, 257), seed + 3).to(dtype)))
        out.append((f"row_{name}_1x16", synth_f32((1, 16), seed + 4).to(dtype)))
        out.append((f"moe_{name}_3x130x260", synth_f32((3, 130, 260), seed + 5).to(dtype)))
        # block (0, 0) all zero, block (0, 1) +-0 only, blocks (1, *) subnormal-sized and tiny values
        x = synth_f32((256, 256), seed + 6)
        x[:128, :128] = 0
        x[:128, 128:] = torch.where(synth_f32((128, 128), seed + 7) < 0, -0.0, 0.0)
        x[128:, :128] = synth_f32((128, 128), seed + 8, spread=0) * torch.finfo(dtype).tiny
        x[128:, 128:] = synth_f32((128, 128), seed + 9, spread=0) * 1e-6
        out.append((f"zeros_subnormals_{name}", x.to(dtype)))
    # bf16 values near 3e38 (the top of bf16's range; 448 / amax stays a normal f32)
    x = (synth_f32((200, 300), 301, spread=0).abs() * 0.4e38 + 2.9e38).to(torch.bfloat16)
    x[::3] = -x[::3]
    out.append(("huge_bfloat16", x))
    # non-finite blocks: +-Inf in block (0, 0), a NaN in block (1, 1), finite blocks beside them
    for k, dtype in enumerate((torch.bfloat16, torch.float32)):
        x = synth_f32((130, 130), 400 + k).to(dtype)
        x[5, 7] = float("inf")
        x[100, 3] = float("-inf")
        x[129, 129] = float("nan")
        out.append((f"nonfinite_{str(dtype).replace('torch.', '')}", x))
    return out


def bits_of(x: torch.Tensor) -> np.ndarray:
    """Raw bits of a bf16/f16 (uint16) or f32 (uint32) tensor."""
    return x.contiguous().view(torch.int16 if x.element_size() == 2 else torch.int32).numpy().view(
        np.uint16 if x.element_size() == 2 else np.uint32)


def digest(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def widen(bits: np.ndarray, dtype: str) -> np.ndarray:
    """Raw source bits (uint16 for bf16/f16, uint32 for f32) -> exact float32 values."""
    if dtype == "bfloat16":
        return (bits.astype(np.uint32) << 16).view(np.float32)
    if dtype == "float16":
        return bits.view(np.float16).astype(np.float32)
    return bits.view(np.float32)


_SRC = {4: ("float16", 2), 5: ("bfloat16", 2), 6: ("float32", 4)}  # TSB_F16, TSB_BF16, TSB_F32


def _host(ptr: int, nbytes: int) -> np.ndarray:
    return np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(ptr))


def replay(blocks: np.ndarray, pieces: np.ndarray) -> None:
    """Execute compiled block/piece tables on host memory: gather each block's pieces, quantise
    it with ``quantize``, store the fp8 rows and the scale."""
    for blk in blocks:
        dtype, es = _SRC[int(blk["src_dtype"])]
        rows, cols = int(blk["rows"]), int(blk["cols"])
        bits = np.zeros((rows, cols), dtype=np.uint16 if es == 2 else np.uint32)
        for p in pieces[int(blk["piece0"]): int(blk["piece0"]) + int(blk["n_pieces"])]:
            pr, pc = int(p["rows"]), int(p["cols"])
            for r in range(pr):
                raw = _host(int(p["src"]) + r * int(p["src_stride"]), pc * es)
                bits[int(p["row0"]) + r, int(p["col0"]): int(p["col0"]) + pc] = raw.view(bits.dtype)
        q, s = quantize(widen(bits, dtype))
        for r in range(rows):
            _host(int(blk["dst"]) + r * int(blk["pitch"]), cols)[:] = q[r]
        _host(int(blk["scale_inv"]), 4)[:] = s.reshape(-1).view(np.uint8)

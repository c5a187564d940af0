"""TEST INFRASTRUCTURE ONLY -- scaled INT8 sources: a bf16/f16/f32 shard at global offset (row0, col0) of its last two
dims quantised into block-, channel- or tensor-scaled symmetric int8 with shard-local groups anchored at the global
origin, and the dequantisation of such int8 shards into bf16/f16/f32.

* ``quantize`` / ``torch_quantize``      int8_oracle's group formula over source_quant_oracle's group cut: per block
                                         the part of a global 128x128 block inside the shard (the shard placed at
                                         (row0 % 128, col0 % 128) of a zero-padded frame: zeros change no group's
                                         max |x|), per channel the shard's part of a row, per tensor its matrix;
* ``dequantize`` / ``torch_dequantize``  ``(q.float() * s_expanded).to(dst)``: f32(q) exact, one float32 multiply,
                                         torch's narrowing;
* ``replay_source`` / ``replay_dequant`` interpreters of the tables ``tsb_source_quant_compile_host_as`` and
                                         ``tsb_dequant_fp8_compile_host`` return, run on host memory with the int8
                                         formats.
"""

from __future__ import annotations

import numpy as np
import torch

from oracle import int8_oracle
from oracle.block_fp8_oracle import BLOCK, bits_of, digest, synth_f32, widen  # noqa: F401  (re-exported for the tests)
from oracle.dequant_fp8_oracle import _DST, _host, expand, narrow, scale_of, scale_shape
from oracle.dequant_fp8_oracle import torch_dequantize as _torch_dequantize
from oracle.source_quant_oracle import _SRC
from oracle.source_quant_oracle import fixture_inputs as quant_inputs  # noqa: F401  (the quantising cases)

GRANULARITIES = ("block", "channel", "tensor")
DSTS = ("bfloat16", "float16", "float32")


def quantize(x: np.ndarray, granularity: str, row0: int = 0, col0: int = 0) -> tuple[np.ndarray, np.ndarray]:
    """x: float32 [..., N, K] (the exactly widened shard) -> (q int8, scale_inv float32 of the shard's groups)."""
    x = np.asarray(x, dtype=np.float32)
    if granularity != "block":
        return int8_oracle.quantize(x, granularity)
    *lead, n, k = x.shape
    ph, pw = row0 % BLOCK, col0 % BLOCK
    frame = np.zeros(tuple(lead) + (ph + n, pw + k), dtype=np.float32)
    frame[..., ph:, pw:] = x
    q, s = int8_oracle.quantize(frame, "block")
    return np.ascontiguousarray(q[..., ph:, pw:]), s


def torch_quantize(x: torch.Tensor, granularity: str, row0: int = 0, col0: int = 0) -> tuple[torch.Tensor, torch.Tensor]:
    """The formula in torch tensor/tensor ops on x's device -> (q int8, scale_inv float32)."""
    if granularity != "block":
        return int8_oracle.torch_quantize(x, granularity)
    ph, pw = row0 % BLOCK, col0 % BLOCK
    frame = torch.nn.functional.pad(x.float(), (pw, 0, ph, 0))
    q, s = int8_oracle.torch_quantize(frame, "block")
    return q[..., ph:, pw:].contiguous(), s


def dequantize(q: np.ndarray, scale: np.ndarray, granularity: str, r0: int = 0, c0: int = 0,
               dst: str = "bfloat16") -> np.ndarray:
    """q: int8 [..., N, K] -> raw bits of the dequantised ``dst`` values."""
    x = np.asarray(q, dtype=np.int8).astype(np.float32)
    with np.errstate(all="ignore"):
        y = (x * expand(scale, x.shape, granularity, r0, c0)).astype(np.float32)
    return narrow(y, dst)


def torch_dequantize(q: torch.Tensor, scale: torch.Tensor, granularity: str, r0: int = 0, c0: int = 0,
                     dst: torch.dtype = torch.bfloat16) -> torch.Tensor:
    """``(q.float() * s_expanded).to(dst)`` on q's device, q int8."""
    assert q.dtype == torch.int8
    return _torch_dequantize(q, scale, granularity, r0, c0, dst)


def assert_invariants(q: np.ndarray, xf: np.ndarray, granularity: str, row0: int = 0, col0: int = 0) -> None:
    """What the formula guarantees in every group of a shard at (row0, col0), whatever its values: no byte is -128,
    a non-finite group is all zeros, and a finite group with amax >= 1e-4 holds +-127 at each of its amax elements."""
    from oracle.ue8m0_oracle import group_amax, group_ids

    gid, n = group_ids(granularity, xf.shape, row0, col0)
    amax = group_amax(xf, gid, n)  # NaN propagates
    finite = np.isfinite(amax)
    assert (q != -128).all(), "a byte is -128"
    assert (q[~finite[gid]] == 0).all(), "a non-finite group holds a non-zero byte"
    big = finite & (amax >= np.float32(1e-4))
    with np.errstate(invalid="ignore"):
        at = big[gid] & (np.abs(xf) == amax[gid])
    assert (np.abs(q[at].astype(np.int16)) == 127).all(), "an amax element is not +-127"
    assert np.array_equal(np.unique(gid[at]), np.flatnonzero(big)), "a finite group lacks its amax element"


def assert_exact(q: torch.Tensor, s: torch.Tensor, x: torch.Tensor, granularity: str, row0: int = 0, col0: int = 0) -> None:
    """int8 q and float32 scale_inv s of a bf16/f16/f32 shard x at (row0, col0): bit for bit the torch rendering on
    q's device and the numpy oracle (bytes exact everywhere, non-finite groups included; scale bits exact,
    NaN-agnostic only where the scale is NaN), and the formula's invariants (``assert_invariants``)."""
    assert q.dtype == torch.int8
    tq, ts = torch_quantize(x.to(q.device), granularity, row0, col0)
    assert torch.equal(q, tq), "int8 bytes differ from the torch rendering"
    got_s = s.cpu().numpy().reshape(-1)
    assert int8_oracle.same_scales(got_s, ts.cpu().numpy().reshape(-1)), "scale_inv differs from the torch rendering"
    xf = widen(bits_of(x.cpu()), str(x.dtype)[6:])
    want_q, want_s = quantize(xf, granularity, row0, col0)
    got_q = q.cpu().numpy()
    assert np.array_equal(got_q, want_q), "int8 bytes differ from the numpy oracle"
    assert int8_oracle.same_scales(got_s, want_s.reshape(-1)), "scale_inv differs from the numpy oracle"
    assert_invariants(got_q, xf, granularity, row0, col0)


def replay_source(units: np.ndarray, tiles: np.ndarray, n_groups: int) -> None:
    """Execute tsb_source_quant_compile_host_as(TSB_I8) tables on host memory: a unit is one group (a block) or
    one group per row (a band); the tiles are the two-pass path, interpreted by int8_oracle.replay_scaled."""
    for u in units:
        dtype, es = _SRC[int(u["src_dtype"])]
        rows, cols = int(u["rows"]), int(u["cols"])
        bits = np.zeros((rows, cols), dtype=np.uint16 if es == 2 else np.uint32)
        for r in range(rows):
            bits[r] = _host(int(u["src"]) + r * int(u["src_pitch"]), cols * es).view(bits.dtype)
        q, s = int8_oracle.quantize(widen(bits, dtype), "channel" if int(u["per_row"]) else "tensor")
        for r in range(rows):
            _host(int(u["dst"]) + r * int(u["dst_pitch"]), cols)[:] = q[r].view(np.uint8)
        s = np.asarray(s, dtype=np.float32).reshape(-1)
        _host(int(u["scale_inv"]), 4 * s.size)[:] = s.view(np.uint8)
    int8_oracle.replay_scaled((), (), tiles, n_groups)


def replay_dequant(tiles: np.ndarray) -> None:
    """Execute tsb_dequant_fp8_compile_host tables of TSB_I8 rects on host memory: every row of a tile reads its
    int8 bytes, multiplies them by the scale at ``scale + r * scale_step`` and stores the narrowed values."""
    for t in tiles:
        dst, es = _DST[int(t["dst_dtype"])]
        rows, cols = int(t["rows"]), int(t["cols"])
        for r in range(rows):
            q = _host(int(t["src"]) + r * int(t["src_stride"]), cols).view(np.int8)
            s = _host(int(t["scale"]) + r * int(t["scale_step"]), 4).view(np.float32)[0]
            with np.errstate(all="ignore"):
                y = (q.astype(np.float32) * s).astype(np.float32)
            _host(int(t["dst"]) + r * int(t["dst_stride"]), cols * es)[:] = narrow(y, dst).view(np.uint8)


def int8_of(shape, seed: int) -> torch.Tensor:
    """Deterministic int8 values over the whole range [-128, 127], rebuilt from an integer hash."""
    x = synth_f32(shape, seed, spread=0)
    return (x.view(torch.int32) & 0xff).to(torch.uint8).view(torch.int8)


# the scale set of the all-values table: every int8 value times each of these (subnormal products, f16 and bf16
# overflow, 0, a negative scale, Inf, NaN)
SCALE_SET = np.array([1.0, 2.0 ** -7, 0.0123 / 127, 2.0 ** -140, 2.0 ** -130, 1000.0, 3e36, 0.0, -0.5, np.inf, np.nan],
                     dtype=np.float32)


def dequant_inputs() -> list[tuple[str, str, int, int, torch.Tensor, torch.Tensor]]:
    """(name, granularity, r0, c0, q, scale) of the dequantising cases: all 256 int8 values per channel against
    SCALE_SET; each granularity on a matrix at an unaligned (r0, c0), an aligned one and an MoE [E, N, K] stack."""
    q = torch.arange(-128, 128, dtype=torch.int16).to(torch.int8).repeat(len(SCALE_SET), 1)
    out = [("all_values", "channel", 0, 0, q, torch.from_numpy(SCALE_SET.copy()).reshape(-1, 1))]
    for k, g in enumerate(GRANULARITIES):
        for name, shape, r0, c0 in (("matrix", (300, 260), 37, 70), ("aligned", (256, 384), 0, 0),
                                    ("moe", (3, 130, 260), 100, 5)):
            seed = 7000 + 100 * k + 10 * len(out)
            out.append((f"{name}_{g}", g, r0, c0, int8_of(shape, seed), scale_of(scale_shape(g, shape, r0, c0), seed + 1)))
    return out

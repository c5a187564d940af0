"""TEST INFRASTRUCTURE ONLY -- power-of-two (UE8M0) scales: the ``scale_fmt="ue8m0"`` variant of every quantising
reference (quantising pulls, requantising pulls, source-side quantisation), on top of the float32 references.

* ``scales_of_amax``       the UE8M0 scale step, a numpy bitwise restatement (the one place the rule lives here);
* ``torch_scales_of_amax`` the same step in torch tensor ops on the integer view of t, on any device (no log2);
* ``quantize`` / ``torch_quantize`` / ``requantize`` / ``torch_requantize``  the references of
  block_fp8_oracle, scaled_fp8_oracle, source_quant_oracle and requant_fp8_oracle with a ``scale_fmt`` option:
  ``None`` is theirs unchanged, ``"ue8m0"`` replaces the scale step;
* ``replay_block`` / ``replay_scaled`` / ``replay_requant`` / ``replay_source``  interpreters of the compiled
  tables of the four quantising kinds with the same option.

The step, per group (the groups are the float32 references' own):
    amax_c    = max(amax, float32(1e-4))                (NaN stays NaN)
    t         = amax_c / 448                             (correctly rounded: the float32 formula's scale_inv)
    scale_inv = t                                        if t's mantissa bits are 0 (a power of two, or Inf)
                (bits(t) & 0x7f800000) + 0x00800000      otherwise (the next power of two up)
    scale     = 1 / scale_inv                            (exact; 0 for Inf)
    q         = e4m3fn(rn(x * scale))
Since t is the float32 references' scale_inv, the variants take it from them and apply the bit rule, then
quantise again with the exact power-of-two scale.  ``ceil(log2(t))`` is not this rule: within float32 rounding of
a power of two it picks one power too small (see ``log2_scale_inv``).
"""

from __future__ import annotations

from collections import defaultdict

import numpy as np
import torch

from oracle import block_fp8_oracle, requant_fp8_oracle, scaled_fp8_oracle, source_quant_oracle
from oracle.block_fp8_oracle import bits_of, digest, synth_f32, widen  # noqa: F401  (re-exported for the tests)
from oracle.dequant_fp8_oracle import dequantize, expand, torch_dequantize
from oracle.scaled_fp8_oracle import _SRC, _gather, _host, narrow

E4M3 = torch.float8_e4m3fn
SCALE_FORMATS = (None, "ue8m0")
GRANULARITIES = ("block", "channel", "tensor")
_CLAMP = np.float32(1e-4)
_FMAX = np.float32(448.0)


def _check(scale_fmt) -> bool:
    if scale_fmt not in SCALE_FORMATS:
        raise ValueError(f"scale_fmt must be one of {SCALE_FORMATS}, not {scale_fmt!r}")
    return scale_fmt == "ue8m0"


def pow2_up(t: np.ndarray) -> np.ndarray:
    """The bit rule on float32 t >= 0: t if its mantissa bits are 0 (or t is NaN), else the next power of two."""
    t = np.asarray(t, dtype=np.float32)
    bits = t.view(np.uint32)
    up = ((bits & np.uint32(0x7F800000)) + np.uint32(0x00800000)).astype(np.uint32)
    out = np.where((bits & np.uint32(0x007FFFFF)) != 0, up, bits).astype(np.uint32).view(np.float32)
    return np.where(np.isnan(t), t, out).astype(np.float32)


def scales_of_amax(amax: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """float32 amax -> (scale, scale_inv) of the UE8M0 step; NaN stays NaN."""
    with np.errstate(all="ignore"):
        amax_c = np.maximum(np.asarray(amax, dtype=np.float32), _CLAMP)  # NaN propagates
        scale_inv = pow2_up((amax_c / _FMAX).astype(np.float32))
        return (np.float32(1.0) / scale_inv).astype(np.float32), scale_inv


def torch_pow2_up(t: torch.Tensor) -> torch.Tensor:
    """``pow2_up`` in torch ops on t's int32 view, on t's device."""
    bits = t.view(torch.int32)
    up = (bits & 0x7F800000) + 0x00800000
    out = torch.where((bits & 0x007FFFFF) != 0, up, bits).view(torch.float32)
    return torch.where(torch.isnan(t), t, out)


def torch_scales_of_amax(amax: torch.Tensor) -> tuple[torch.Tensor, torch.Tensor]:
    """The UE8M0 step in torch tensor/tensor ops -> (scale, scale_inv), float32 on amax's device."""
    amax_c = torch.maximum(amax.float(), torch.full_like(amax.float(), 1e-4))
    scale_inv = torch_pow2_up(amax_c.div(torch.full_like(amax_c, 448.0)))
    return torch.ones_like(scale_inv).div(scale_inv), scale_inv


def log2_scale_inv(t: np.ndarray) -> np.ndarray:
    """``2 ** ceil(log2(t))`` as some libraries write the step, in float32 (for the tests: where it differs)."""
    t = np.asarray(t, dtype=np.float32)
    with np.errstate(all="ignore"):
        return np.exp2(np.ceil(np.log2(t))).astype(np.float32)


# ---- the quantising references with scale_fmt ----------------------------------------------------------------
def _base(x: np.ndarray, granularity: str, row0: int, col0: int) -> tuple[np.ndarray, np.ndarray]:
    if granularity not in GRANULARITIES:
        raise ValueError(f"granularity must be one of {GRANULARITIES}, not {granularity!r}")
    if row0 or col0:
        return source_quant_oracle.quantize(x, granularity, row0, col0)
    if granularity == "block":
        return block_fp8_oracle.quantize(x)
    return scaled_fp8_oracle.quantize(x, granularity)


def quantize(x: np.ndarray, granularity: str, row0: int = 0, col0: int = 0,
             scale_fmt: str | None = None) -> tuple[np.ndarray, np.ndarray]:
    """x: float32 [..., N, K] (exactly widened) -> (q uint8, scale_inv float32) with groups of ``granularity``,
    shard-local and anchored at the global origin for a shard at (row0, col0) (block_fp8_oracle /
    scaled_fp8_oracle at (0, 0), source_quant_oracle elsewhere)."""
    x = np.asarray(x, dtype=np.float32)
    q, t = _base(x, granularity, row0, col0)
    if not _check(scale_fmt):
        return q, t
    scale_inv = pow2_up(t)
    with np.errstate(all="ignore"):
        scale = (np.float32(1.0) / scale_inv).astype(np.float32)
        prod = (x * expand(scale, x.shape, granularity, row0, col0)).astype(np.float32)
    return narrow(prod), scale_inv


def torch_quantize(x: torch.Tensor, granularity: str, row0: int = 0, col0: int = 0,
                   scale_fmt: str | None = None) -> tuple[torch.Tensor, torch.Tensor]:
    """``quantize`` in torch tensor/tensor ops on x's device -> (q float8_e4m3fn, scale_inv float32)."""
    if granularity not in GRANULARITIES:
        raise ValueError(f"granularity must be one of {GRANULARITIES}, not {granularity!r}")
    q, t = source_quant_oracle.torch_quantize(x, granularity, row0, col0)
    if not _check(scale_fmt):
        return q, t
    xf = x.float()
    *lead, n, k = xf.shape
    scale_inv = torch_pow2_up(t)
    scale = torch.ones_like(scale_inv).div(scale_inv)
    if granularity == "block":
        gr = torch.div(row0 + torch.arange(n, device=xf.device), 128, rounding_mode="floor") - row0 // 128
        gc = torch.div(col0 + torch.arange(k, device=xf.device), 128, rounding_mode="floor") - col0 // 128
        full = scale[..., gr[:, None], gc[None, :]]
    elif granularity == "channel":
        full = scale
    else:
        full = scale.reshape(*lead, 1, 1)
    return xf.mul(full).to(E4M3), scale_inv


def requantize(q: np.ndarray, scale: np.ndarray, src_g: str, r0: int, c0: int, dst_g: str,
               scale_fmt: str | None = None) -> tuple[np.ndarray, np.ndarray]:
    """requant_fp8_oracle.requantize with the destination's scale step chosen by ``scale_fmt``."""
    x = dequantize(q, scale, src_g, r0, c0, "float32").view(np.float32)
    return quantize(x, dst_g, scale_fmt=scale_fmt)


def torch_requantize(q: torch.Tensor, scale: torch.Tensor, src_g: str, r0: int, c0: int, dst_g: str,
                     scale_fmt: str | None = None) -> tuple[torch.Tensor, torch.Tensor]:
    """requant_fp8_oracle.torch_requantize with the destination's scale step chosen by ``scale_fmt``."""
    x = torch_dequantize(q, scale, src_g, r0, c0, torch.float32)
    return torch_quantize(x, dst_g, scale_fmt=scale_fmt)


def fixture_inputs() -> list[tuple[str, torch.Tensor, str, int, int]]:
    """The cases of tests/golden/ue8m0_vectors.npz as (name, x, granularity, row0, col0): random bf16/f16/f32
    [300, 200] matrices and a [3, 130, 260] stack, per block, channel and tensor at (0, 0) (the quantising pulls'
    groups) and at (37, 70) (shard-local source groups anchored at the global origin); a float32 matrix whose
    rows hit the step's edges (amax 0, 1e-5, 448 * 2^k exactly, one ulp above, just below 448 * 2^(k+1), FLT_MAX),
    and a bf16 matrix with an Inf row and a NaN row."""
    out = []
    for k, dtype in enumerate((torch.bfloat16, torch.float16, torch.float32)):
        name = str(dtype).replace("torch.", "")
        for gi, g in enumerate(GRANULARITIES):
            seed = 9000 + 100 * k + 10 * gi
            for r0, c0 in ((0, 0), (37, 70)):
                out.append((f"{g}_{name}_300x200_at_{r0}_{c0}", synth_f32((300, 200), seed + r0).to(dtype), g, r0, c0))
            out.append((f"{g}_{name}_moe_3x130x260", synth_f32((3, 130, 260), seed + 5).to(dtype), g, 0, 0))
    edges = edge_matrix()
    special = synth_f32((260, 140), 9901).to(torch.bfloat16)
    special[3, 5] = float("inf")
    special[200, 100] = float("nan")
    for g in GRANULARITIES:
        out.append((f"{g}_float32_edges", edges, g, 0, 0))
        out.append((f"{g}_bfloat16_nonfinite", special, g, 0, 0))
        out.append((f"{g}_bfloat16_nonfinite_at_37_70", special, g, 37, 70))
    return out


def edge_amaxes() -> np.ndarray:
    """float32 amax values on the step's edges: 0, 1e-5 (clamped), 448 * 2^k, 448 * 2^k * (1 + 2^-23), the float
    just below 448 * 2^(k+1), and FLT_MAX."""
    vals = [0.0, 1e-5]
    for k in (-20, -8, -1, 0, 1, 7, 40, 100):
        base = np.float32(448.0 * 2.0 ** k)
        vals += [base, np.nextafter(base, np.float32(np.inf)), np.nextafter(np.float32(2 * base), np.float32(0))]
    vals.append(np.finfo(np.float32).max)
    return np.array(vals, dtype=np.float32)


def edge_matrix() -> torch.Tensor:
    """A float32 [len(edge_amaxes()), 160] matrix: row i holds edge_amaxes()[i] once (at column 7 + i) among
    smaller values of both signs, so per channel its amax is that edge."""
    a = edge_amaxes()
    x = synth_f32((a.size, 160), 9902, spread=0).numpy() * 0.5
    x = (x * a[:, None]).astype(np.float32)
    for i, v in enumerate(a):
        x[i, 7 + i] = -v if i % 2 else v
    return torch.from_numpy(x)


# ---- table replayers with scale_fmt --------------------------------------------------------------------------
def _quantize_group(x: np.ndarray, per_row: bool, scale_fmt) -> tuple[np.ndarray, np.ndarray]:
    """One group (the whole of x) or one per row."""
    return quantize(x, "channel" if per_row else "tensor", scale_fmt=scale_fmt)


def _store(dst: int, pitch: int, q: np.ndarray) -> None:
    for r in range(q.shape[0]):
        _host(dst + r * pitch, q.shape[1])[:] = q[r]


def _store_scales(addr: int, s: np.ndarray) -> None:
    s = np.ascontiguousarray(s, dtype=np.float32).reshape(-1)
    _host(addr, 4 * s.size)[:] = s.view(np.uint8)


def _replay_tiles(tiles: np.ndarray, values: list, n_groups: int, scale_fmt) -> None:
    """Two-pass tiles: each group's amax over its tiles, then every tile quantised with its group's scale."""
    ue8m0 = _check(scale_fmt)
    amax = defaultdict(lambda: np.float32(0))
    for t, x in zip(tiles, values):
        g = int(t["group"])
        assert g < n_groups
        amax[g] = np.maximum(amax[g], np.abs(x).max())  # NaN propagates
    for t, x in zip(tiles, values):
        scale, scale_inv = (scales_of_amax if ue8m0 else scaled_fp8_oracle.scales_of_amax)(amax[int(t["group"])])
        with np.errstate(all="ignore"):
            _store(int(t["dst"]), int(t["pitch"]), narrow((x * scale).astype(np.float32)))
        if int(t["scale_inv"]):
            _store_scales(int(t["scale_inv"]), np.asarray(scale_inv))


def _src_tile(t) -> np.ndarray:
    dtype, es = _SRC[int(t["src_dtype"])]
    return widen(_gather(int(t["src"]), int(t["src_stride"]), int(t["rows"]), int(t["cols"]), es), dtype)


def _pieces_bits(rows: int, cols: int, es: int, pieces) -> np.ndarray:
    bits = np.zeros((rows, cols), dtype=np.uint16 if es == 2 else np.uint32)
    for p in pieces:
        r0, c0, pr, pc = (int(p[f]) for f in ("row0", "col0", "rows", "cols"))
        bits[r0: r0 + pr, c0: c0 + pc] = _gather(int(p["src"]), int(p["src_stride"]), pr, pc, es)
    return bits


def replay_block(blocks: np.ndarray, pieces: np.ndarray, scale_fmt: str | None = None) -> None:
    """block_fp8_oracle.replay with ``scale_fmt``: each block is one group."""
    for blk in blocks:
        dtype, es = _SRC[int(blk["src_dtype"])]
        first = int(blk["piece0"])
        x = widen(_pieces_bits(int(blk["rows"]), int(blk["cols"]), es, pieces[first: first + int(blk["n_pieces"])]), dtype)
        q, s = _quantize_group(x, False, scale_fmt)
        _store(int(blk["dst"]), int(blk["pitch"]), q)
        _store_scales(int(blk["scale_inv"]), s)


def replay_scaled(bands: np.ndarray, pieces: np.ndarray, tiles: np.ndarray, n_groups: int,
                  scale_fmt: str | None = None) -> None:
    """scaled_fp8_oracle.replay with ``scale_fmt``: bands one group per row, tiles two-pass."""
    for b in bands:
        dtype, es = _SRC[int(b["src_dtype"])]
        first = int(b["piece0"])
        x = widen(_pieces_bits(int(b["rows"]), int(b["cols"]), es, pieces[first: first + int(b["n_pieces"])]), dtype)
        q, s = _quantize_group(x, True, scale_fmt)
        _store(int(b["dst"]), int(b["cols"]), q)
        _store_scales(int(b["scale_inv"]), s)
    _replay_tiles(tiles, [_src_tile(t) for t in tiles], n_groups, scale_fmt)


def replay_source(units: np.ndarray, tiles: np.ndarray, n_groups: int, scale_fmt: str | None = None) -> None:
    """source_quant_oracle.replay with ``scale_fmt``: units one group (a block) or one per row, tiles two-pass."""
    for u in units:
        dtype, es = _SRC[int(u["src_dtype"])]
        x = widen(_gather(int(u["src"]), int(u["src_pitch"]), int(u["rows"]), int(u["cols"]), es), dtype)
        q, s = _quantize_group(x, bool(int(u["per_row"])), scale_fmt)
        _store(int(u["dst"]), int(u["dst_pitch"]), q)
        _store_scales(int(u["scale_inv"]), s)
    _replay_tiles(tiles, [_src_tile(t) for t in tiles], n_groups, scale_fmt)


def replay_requant(units: np.ndarray, pieces: np.ndarray, tiles: np.ndarray, n_groups: int,
                   scale_fmt: str | None = None) -> None:
    """requant_fp8_oracle.replay with ``scale_fmt``: units one group (a block) or one per row, tiles two-pass."""
    x_of = requant_fp8_oracle._x
    for u in units:
        rows, cols = int(u["rows"]), int(u["cols"])
        x = np.full((rows, cols), np.nan, dtype=np.float32)
        for p in pieces[int(u["piece0"]): int(u["piece0"]) + int(u["n_pieces"])]:
            r0, c0, pr, pc = (int(p[f]) for f in ("row0", "col0", "rows", "cols"))
            x[r0: r0 + pr, c0: c0 + pc] = x_of(int(p["src"]), int(p["src_stride"]), int(p["scale"]), int(p["scale_step"]), pr,
                                               pc, int(p["col_phase"]), int(p["col_blocks"]))
        q, s = _quantize_group(x, bool(int(u["per_row"])), scale_fmt)
        _store(int(u["dst"]), int(u["pitch"]), q)
        _store_scales(int(u["scale_inv"]), s)
    values = [x_of(int(t["src"]), int(t["src_stride"]), int(t["scale"]), int(t["scale_step"]), int(t["rows"]), int(t["cols"]))
              for t in tiles]
    _replay_tiles(tiles, values, n_groups, scale_fmt)

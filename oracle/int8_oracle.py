"""TEST INFRASTRUCTURE ONLY -- symmetric INT8 destinations of the quantising pulls: the formula group by group in
numpy, its torch rendering, interpreters of the compiled block / band / tile tables, and the fixture inputs.

Per group (a 128x128 block anchored at the matrix's (0, 0), edge blocks partial; one row; or the whole matrix;
leading dims are independent matrices), x widened exactly to float32:
    amax      = max |x| over the group                    (NaN if any element is NaN)
    amax_c    = max(amax, float32(1e-4))                  (NaN stays NaN)
    scale     = 127 / amax_c ;  scale_inv = amax_c / 127  (IEEE float32 division, round to nearest even)
    q         = int8(sat[-128, 127](rne_int(rn_f32(x * scale))))  with NaN -> 0
A NaN group gets scale_inv NaN and q = 0; an Inf group scale 0, scale_inv Inf and q = 0 (Inf * 0 is NaN).
"""

from __future__ import annotations

from collections import defaultdict

import numpy as np
import torch

from oracle.block_fp8_oracle import bits_of, digest, synth_f32, widen  # noqa: F401  (re-exported for the tests)
from oracle.scaled_fp8_oracle import _SRC, _gather, _host

GRANULARITIES = ("block", "channel", "tensor")
BLOCK = 128
_CLAMP = np.float32(1e-4)
_QMAX = np.float32(127.0)


def scales_of_amax(amax) -> tuple[np.ndarray, np.ndarray]:
    """float32 amax -> (scale, scale_inv), float32; NaN stays NaN, Inf gives (0, Inf)."""
    with np.errstate(all="ignore"):
        amax_c = np.maximum(np.asarray(amax, dtype=np.float32), _CLAMP)  # NaN propagates
        return (_QMAX / amax_c).astype(np.float32), (amax_c / _QMAX).astype(np.float32)


def narrow(x: np.ndarray, scale) -> np.ndarray:
    """float32 x -> int8 q with one group scale: rn_f32(x * scale), round half to even, NaN -> 0, saturated."""
    with np.errstate(all="ignore"):
        prod = (np.asarray(x, dtype=np.float32) * np.float32(scale)).astype(np.float32)
        r = np.rint(prod)
    r[np.isnan(r)] = 0
    return np.clip(r, -128, 127).astype(np.int8)


def quantize_group(x: np.ndarray) -> tuple[np.ndarray, np.float32]:
    """One group (the whole of x) -> (q int8, scale_inv)."""
    with np.errstate(all="ignore"):
        amax = np.abs(np.asarray(x, dtype=np.float32)).max() if x.size else np.float32(0)  # NaN propagates
    scale, scale_inv = scales_of_amax(amax)
    return narrow(x, scale), np.float32(scale_inv)


def scale_shape(granularity: str, shape) -> tuple:
    """The float32 scale_inv tensor of an int8 destination of ``shape``: lead + (ceil(N/128), ceil(K/128)) per
    block, lead + (N, 1) per channel, lead per tensor."""
    *lead, n, k = shape
    return {"block": (*lead, -(-n // BLOCK), -(-k // BLOCK)), "channel": (*lead, n, 1), "tensor": tuple(lead)}[granularity]


def quantize(x: np.ndarray, granularity: str) -> tuple[np.ndarray, np.ndarray]:
    """x: float32 [..., N, K] -> (q int8 [..., N, K], scale_inv float32 of ``scale_shape``), group by group."""
    if granularity not in GRANULARITIES:
        raise ValueError(f"granularity must be one of {GRANULARITIES}, not {granularity!r}")
    x = np.asarray(x, dtype=np.float32)
    *lead, n, k = x.shape
    q = np.zeros(x.shape, dtype=np.int8)
    s = np.zeros(scale_shape(granularity, x.shape), dtype=np.float32)
    for li in np.ndindex(*lead):
        m, qm, sm = x[li], q[li], s[li]
        if granularity == "block":
            for br in range(-(-n // BLOCK)):
                for bc in range(-(-k // BLOCK)):
                    blk = (slice(br * BLOCK, (br + 1) * BLOCK), slice(bc * BLOCK, (bc + 1) * BLOCK))
                    qm[blk], sm[br, bc] = quantize_group(m[blk])
        elif granularity == "channel":
            for r in range(n):
                qm[r], sm[r, 0] = quantize_group(m[r])
        else:
            qm[...], s[li] = quantize_group(m)
    return q, s


def torch_quantize(x: torch.Tensor, granularity: str) -> tuple[torch.Tensor, torch.Tensor]:
    """The formula in torch tensor/tensor ops on x's device -> (q int8, scale_inv float32 of ``scale_shape``):
    ``torch.round(xf * scale).nan_to_num(nan=0.0).clamp(-128, 127).to(torch.int8)``."""
    if granularity not in GRANULARITIES:
        raise ValueError(f"granularity must be one of {GRANULARITIES}, not {granularity!r}")
    xf = x.float()
    *lead, n, k = xf.shape
    a = xf.abs()
    if granularity == "block":
        nb, kb = -(-n // BLOCK), -(-k // BLOCK)
        a = torch.nn.functional.pad(a, (0, kb * BLOCK - k, 0, nb * BLOCK - n))
        amax = a.reshape(*lead, nb, BLOCK, kb, BLOCK).amax(dim=(-3, -1))
    elif granularity == "channel":
        amax = a.amax(dim=-1, keepdim=True)
    else:
        amax = a.reshape(*lead, n * k).amax(dim=-1)
    amax_c = torch.maximum(amax, torch.full_like(amax, 1e-4))
    scale = torch.full_like(amax_c, 127.0).div(amax_c)
    scale_inv = amax_c.div(torch.full_like(amax_c, 127.0))
    if granularity == "block":
        gr = torch.arange(n, device=xf.device) // BLOCK
        gc = torch.arange(k, device=xf.device) // BLOCK
        full = scale[..., gr[:, None], gc[None, :]]
    elif granularity == "channel":
        full = scale
    else:
        full = scale.reshape(*lead, 1, 1)
    q = torch.round(xf * full).nan_to_num(nan=0.0).clamp(-128, 127).to(torch.int8)
    return q, scale_inv


# ---- table replayers: the compiled block / band / tile tables executed on host memory with the int8 formula -----
def _store(dst: int, pitch: int, q: np.ndarray) -> None:
    for r in range(q.shape[0]):
        _host(dst + r * pitch, q.shape[1])[:] = q[r].view(np.uint8)


def _store_scales(addr: int, s) -> None:
    s = np.ascontiguousarray(s, dtype=np.float32).reshape(-1)
    _host(addr, 4 * s.size)[:] = s.view(np.uint8)


def _pieces(rows: int, cols: int, src_dtype: int, pieces) -> np.ndarray:
    dtype, es = _SRC[src_dtype]
    bits = np.zeros((rows, cols), dtype=np.uint16 if es == 2 else np.uint32)
    for p in pieces:
        r0, c0, pr, pc = (int(p[f]) for f in ("row0", "col0", "rows", "cols"))
        bits[r0: r0 + pr, c0: c0 + pc] = _gather(int(p["src"]), int(p["src_stride"]), pr, pc, es)
    return widen(bits, dtype)


def replay_block(blocks: np.ndarray, pieces: np.ndarray) -> None:
    """tsb_block_fp8_compile_host's tables with TSB_I8 rects: each block one group."""
    for blk in blocks:
        first = int(blk["piece0"])
        x = _pieces(int(blk["rows"]), int(blk["cols"]), int(blk["src_dtype"]), pieces[first: first + int(blk["n_pieces"])])
        q, s = quantize_group(x)
        _store(int(blk["dst"]), int(blk["pitch"]), q)
        _store_scales(int(blk["scale_inv"]), s)


def replay_scaled(bands: np.ndarray, pieces: np.ndarray, tiles: np.ndarray, n_groups: int) -> None:
    """tsb_scaled_fp8_compile_host's tables with TSB_I8 rects: bands one group per row; tiles two-pass (each
    group's amax over its tiles, then every tile with its group's scale; the designated tile stores scale_inv)."""
    for b in bands:
        first = int(b["piece0"])
        x = _pieces(int(b["rows"]), int(b["cols"]), int(b["src_dtype"]), pieces[first: first + int(b["n_pieces"])])
        for r in range(x.shape[0]):
            q, s = quantize_group(x[r])
            _store(int(b["dst"]) + r * int(b["cols"]), int(b["cols"]), q[None])
            _store_scales(int(b["scale_inv"]) + 4 * r, s)
    values = []
    for t in tiles:
        dtype, es = _SRC[int(t["src_dtype"])]
        values.append(widen(_gather(int(t["src"]), int(t["src_stride"]), int(t["rows"]), int(t["cols"]), es), dtype))
    amax = defaultdict(lambda: np.float32(0))
    for t, x in zip(tiles, values):
        g = int(t["group"])
        assert g < n_groups
        with np.errstate(all="ignore"):
            amax[g] = np.maximum(amax[g], np.abs(x).max())  # NaN propagates
    for t, x in zip(tiles, values):
        scale, scale_inv = scales_of_amax(amax[int(t["group"])])
        _store(int(t["dst"]), int(t["pitch"]), narrow(x, scale))
        if int(t["scale_inv"]):
            _store_scales(int(t["scale_inv"]), scale_inv)


# ---- fixture inputs ----------------------------------------------------------------------------------------------
SPECIALS = ("ties", "zero", "nan", "inf", "nan_inf", "max", "subnormal")
_MAX = {torch.bfloat16: torch.finfo(torch.bfloat16).max, torch.float16: torch.finfo(torch.float16).max,
        torch.float32: torch.finfo(torch.float32).max}


def _plant(m: torch.Tensor, values: list) -> None:
    """Put ``values`` into every row of m once per 128-column block (at shifting columns), so that every row,
    every block and the matrix hold each of them (the first wins where a narrow edge block has too few columns)."""
    n, k = m.shape
    for r in range(n):
        for c0 in range(0, k, BLOCK):
            w = min(BLOCK, k - c0)
            for j, v in reversed(list(enumerate(values))):
                m[r, c0 + (r + j) % w] = v


def special_stack(dtype: torch.dtype, shape=(130, 260)) -> torch.Tensor:
    """A [len(SPECIALS), N, K] stack of ``dtype``, matrix i holding special i in every row, block and matrix:
    ties  k + 1/2 steps with 127 as the amax (scale exactly 1: every product is a tie or an integer);
    zero  all zeros (the 1e-4 floor);  nan / inf / nan_inf  NaN, +-Inf or both among random values;
    max   the dtype's largest finite value among random values;  subnormal  only subnormal values of ``dtype``."""
    n, k = shape
    out = []
    rnd = synth_f32((len(SPECIALS), n, k), 8801)
    for i, name in enumerate(SPECIALS):
        m = rnd[i].clone()
        if name == "ties":
            steps = torch.floor(rnd[i] * 127).clamp(-127, 126)
            m = steps + 0.5
            _plant(m, [127.0, -126.5, 0.5, -0.5, 1.5, -2.5])
        elif name == "zero":
            m = torch.zeros(n, k)
        elif name == "nan":
            _plant(m, [float("nan")])
        elif name == "inf":
            _plant(m, [float("inf"), float("-inf")])
        elif name == "nan_inf":
            _plant(m, [float("nan"), float("inf")])
        elif name == "max":
            m = m.to(dtype)
            _plant(m, [_MAX[dtype], -_MAX[dtype]])
        elif name == "subnormal":
            tiny = torch.finfo(dtype).smallest_normal
            m = (rnd[i] * tiny).to(dtype)
            m[m.abs() >= tiny] = 0
        out.append(m.to(dtype))
    return torch.stack(out)


def fixture_inputs() -> list[tuple[str, torch.Tensor, str]]:
    """The cases of tests/golden/int8_vectors.npz as (name, x, granularity): per granularity and bf16/f16/f32 source
    a random [300, 200] matrix (partial edge blocks), a random [3, 130, 260] MoE stack and the special stack."""
    out = []
    for k, dtype in enumerate((torch.bfloat16, torch.float16, torch.float32)):
        name = str(dtype).replace("torch.", "")
        special = special_stack(dtype)
        for gi, g in enumerate(GRANULARITIES):
            seed = 8000 + 100 * k + 10 * gi
            out.append((f"{g}_{name}_300x200", synth_f32((300, 200), seed).to(dtype), g))
            out.append((f"{g}_{name}_moe_3x130x260", synth_f32((3, 130, 260), seed + 5).to(dtype), g))
            out.append((f"{g}_{name}_special_{len(SPECIALS)}x130x260", special, g))
    return out


def same_scales(a: np.ndarray, b: np.ndarray) -> bool:
    """float32 scales equal bit for bit, NaN-agnostically (NaN bit patterns are the platform's)."""
    a, b = np.asarray(a, dtype=np.float32), np.asarray(b, dtype=np.float32)
    if a.shape != b.shape or not np.array_equal(np.isnan(a), np.isnan(b)):
        return False
    fin = ~np.isnan(a)
    return np.array_equal(a[fin].view(np.uint32), b[fin].view(np.uint32))

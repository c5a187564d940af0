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

import functools
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


# ---- edge values of the scale step: inputs that tell the formula from plausible wrong renderings of it ----------
# Each rendering maps (float32 x, the group's float32 scale and scale_inv) to the integer before the NaN rule and the
# saturation; RENDERINGS[0] is the formula, the others are slips a kernel could make.
RENDERINGS = ("formula", "div_scale_inv", "mul_rcp_scale_inv", "unrounded_product", "half_away_from_zero", "truncation")
WRONG = RENDERINGS[1:]


def render(name: str, x: np.ndarray, scale, scale_inv) -> np.ndarray:
    """x (float32) -> int8 by rendering ``name``, with the NaN rule and saturation of ``narrow``:
    formula              rint(rn_f32(x * scale))
    div_scale_inv        rint(rn_f32(x / scale_inv))
    mul_rcp_scale_inv    rint(rn_f32(x * rn_f32(1 / scale_inv)))
    unrounded_product    rint(x * scale in float64)
    half_away_from_zero  rn_f32(x * scale) rounded half away from zero
    truncation           rn_f32(x * scale) truncated toward zero"""
    x = np.asarray(x, dtype=np.float32)
    scale, scale_inv = np.float32(scale), np.float32(scale_inv)
    with np.errstate(all="ignore"):
        prod = (x * scale).astype(np.float32)
        if name == "formula":
            r = np.rint(prod)
        elif name == "div_scale_inv":
            r = np.rint((x / scale_inv).astype(np.float32))
        elif name == "mul_rcp_scale_inv":
            r = np.rint((x * (np.float32(1) / scale_inv).astype(np.float32)).astype(np.float32))
        elif name == "unrounded_product":
            r = np.rint(x.astype(np.float64) * np.float64(scale))
        elif name == "half_away_from_zero":
            p = prod.astype(np.float64)
            r = np.sign(p) * np.floor(np.abs(p) + 0.5)
        elif name == "truncation":
            r = np.trunc(prod)
        else:
            raise ValueError(f"rendering must be one of {RENDERINGS}, not {name!r}")
    r = np.where(np.isnan(r), 0, r)
    return np.clip(r, -128, 127).astype(np.int8)


def discriminated(x: np.ndarray, amax) -> dict[str, np.ndarray]:
    """{wrong rendering: mask of the elements of x where it gives another byte than the formula}, for a group of
    max |x| ``amax`` (broadcast: one amax per element is fine)."""
    x = np.asarray(x, dtype=np.float32)
    amax = np.broadcast_to(np.asarray(amax, dtype=np.float32), x.shape)
    out = {n: np.zeros(x.shape, dtype=bool) for n in WRONG}
    for a in np.unique(amax):
        sel = amax == a
        scale, scale_inv = scales_of_amax(a)
        want = render("formula", x[sel], scale, scale_inv)
        for n in WRONG:
            out[n][sel] = render(n, x[sel], scale, scale_inv) != want
    return out


def tie_kinds(x: np.ndarray, amax) -> set:
    """{(k parity "even"/"odd", sign +1/-1)} of the elements whose rounded product x * scale is exactly k + 1/2."""
    x = np.asarray(x, dtype=np.float32)
    scale, _ = scales_of_amax(np.broadcast_to(np.asarray(amax, dtype=np.float32), x.shape))
    with np.errstate(all="ignore"):
        p = (x * scale).astype(np.float32).astype(np.float64)
    tie = np.isfinite(p) & (np.abs(p) - np.floor(np.abs(p)) == 0.5)
    k = np.floor(np.abs(p[tie])).astype(np.int64)
    return {("even" if kk % 2 == 0 else "odd", 1 if s > 0 else -1) for kk, s in zip(k, p[tie])}


_TOP_BITS = {"bfloat16": 0x7F80, "float16": 0x7C00}  # the first non-finite bit pattern


@functools.lru_cache(maxsize=None)
def _positive_values(dtype: str) -> np.ndarray:
    """Every positive finite value of a 2-byte float dtype, widened to float32, ascending."""
    return widen(np.arange(1, _TOP_BITS[dtype], dtype=np.uint16), dtype)


def edge_values(dtype: str, amax) -> np.ndarray:
    """The positive values of ``dtype`` up to ``amax`` (itself a ``dtype`` value) at which some wrong rendering
    differs from the formula, for a group of that amax: every finite bf16 / f16 value is tried; for float32, 8 ulps
    either side of each (k + 1/2) / scale."""
    a = np.float32(amax)
    scale, scale_inv = scales_of_amax(a)
    if dtype == "float32":
        centre = ((np.arange(128) + 0.5) / np.float64(scale)).astype(np.float32)
        cand = [centre]
        up, down = centre.copy(), centre.copy()
        for _ in range(8):
            up, down = np.nextafter(up, np.float32(np.inf)), np.nextafter(down, np.float32(0))
            cand += [up, down]
        cand = np.unique(np.concatenate(cand))
    else:
        cand = _positive_values(dtype)
    cand = cand[(cand > 0) & (cand <= a)]
    told = discriminated(cand, a)
    hard = np.any([told[n] for n in HARD], axis=0)
    # the values that tell a HARD rendering apart first, then the ties k + 1/2, then the rest
    p = (cand * scale).astype(np.float32).astype(np.float64)
    rank = np.where(hard, 0, np.where(p - np.floor(p) == 0.5, 1, 2))
    hit = np.any(list(told.values()), axis=0)
    return cand[hit][np.argsort(rank[hit], kind="stable")]


HARD = ("div_scale_inv", "mul_rcp_scale_inv", "unrounded_product")  # the renderings few values tell apart


def clamp_amaxes(dtype: str) -> np.ndarray:
    """Three amaxes at the 1e-4 floor in ``dtype``: for float32 the values just below, at and just above 1e-4f; for
    bf16 / f16 (which do not hold 1e-4f) its two largest values below 1e-4f and its smallest one above."""
    if dtype == "float32":
        return np.array([np.nextafter(_CLAMP, np.float32(0)), _CLAMP, np.nextafter(_CLAMP, np.float32(1))], dtype=np.float32)
    v = _positive_values(dtype)
    i = int(np.searchsorted(v, _CLAMP))  # v[i - 1] < 1e-4f <= v[i]; neither dtype holds 1e-4f exactly
    assert v[i] > _CLAMP
    return np.array([v[i - 2], v[i - 1], v[i]], dtype=np.float32)


@functools.lru_cache(maxsize=None)
def edge_groups(dtype: str, n: int = 12) -> tuple:
    """(amax, edge values) of the groups an edge input plants in ``dtype``: the three clamp_amaxes, 127 (scale exactly
    1: the ties k + 1/2), then ``n`` amaxes searched from a log-uniform sequence over [2^-6, 2^8], picked so that each
    rendering of HARD is told apart in at least two of them."""
    out = [(a, edge_values(dtype, a)) for a in clamp_amaxes(dtype)] + [(np.float32(127), edge_values(dtype, np.float32(127)))]
    rng = np.random.default_rng({"bfloat16": 1, "float16": 2, "float32": 3}[dtype])
    need = {h: 2 for h in HARD}
    spare = []
    for _ in range(4000):
        if len(out) == n + 4:
            break
        a = np.float32(2.0 ** rng.uniform(-6, 8))
        a = widen(bits_of(torch.tensor(float(a)).to(getattr(torch, dtype))), dtype)[()]
        vals = edge_values(dtype, a)
        if not len(vals):
            continue
        told = {h for h, m in discriminated(vals, a).items() if h in HARD and m.any()}
        if any(need[h] > 0 for h in told):
            for h in told:
                need[h] -= 1
            out.append((a, vals))
        elif len(spare) < n:
            spare.append((a, vals))
    out += spare[: n + 4 - len(out)]
    assert len(out) == n + 4 and all(v <= 0 for v in need.values()), (dtype, need)
    return tuple(out)


def plant_rounding_edges(shape, dtype: torch.dtype, granularity: str, row0: int = 0, col0: int = 0):
    """A ``dtype`` shard whose groups (anchored as the granularity's, at (row0, col0)) take edge_groups(dtype) in
    turn: the amax, negated in odd groups, at the group's first element, then the group's edge values in turn as
    +v, -v.  Groups past the last edge group repeat them from the first.  -> (x, number of groups)."""
    from oracle.ue8m0_oracle import group_ids

    name = str(dtype)[6:]
    groups = edge_groups(name)
    gid, n = group_ids(granularity, shape, row0, col0)
    flat_gid = gid.reshape(-1)
    x = np.zeros(flat_gid.shape, dtype=np.float32)
    order = np.argsort(flat_gid, kind="stable")
    starts = np.searchsorted(flat_gid[order], np.arange(n + 1))
    for g in range(n):
        idx = order[starts[g]: starts[g + 1]]
        a, vals = groups[g % len(groups)]
        seq = np.stack([vals, -vals], axis=1).reshape(-1)
        fill = np.resize(seq, max(0, idx.size - 1)) if seq.size else np.zeros(max(0, idx.size - 1), np.float32)
        x[idx[1:]] = fill
        x[idx[0]] = -a if g % 2 else a
    return torch.from_numpy(x.reshape(tuple(shape))).to(dtype), n


def told_apart(x: torch.Tensor, granularity: str, row0: int = 0, col0: int = 0) -> tuple[set, set]:
    """From a shard's values alone: (the wrong renderings that give another byte than the formula somewhere in it,
    the tie kinds of tie_kinds over it), each element with its own group's amax."""
    from oracle.ue8m0_oracle import group_amax, group_ids

    xf = widen(bits_of(x), str(x.dtype)[6:])
    gid, n = group_ids(granularity, tuple(x.shape), row0, col0)
    amax = group_amax(xf, gid, n)[gid]
    told = {name for name, m in discriminated(xf, amax).items() if m.any()}
    return told, tie_kinds(xf, amax)


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

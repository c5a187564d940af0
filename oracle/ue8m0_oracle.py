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


# ---- inputs on the step's edges, power-of-two source scales and checks -----------------------------------------
BRANCHES = ("keep", "up", "clamp")


def branch_of_amax(amax: np.ndarray) -> np.ndarray:
    """The branch of the step each finite amax takes: "clamp" below 1e-4 (zero and subnormal groups included),
    "keep" where t = amax / 448 is a power of two, "up" elsewhere."""
    amax = np.asarray(amax, dtype=np.float32)
    with np.errstate(all="ignore"):
        t = (np.maximum(amax, _CLAMP) / _FMAX).astype(np.float32)
    keep = (t.view(np.uint32) & np.uint32(0x007FFFFF)) == 0
    return np.where(amax < _CLAMP, "clamp", np.where(keep, "keep", "up"))


def group_amax(x: np.ndarray, gid: np.ndarray, n_groups: int) -> np.ndarray:
    """max |x| per group id (x float32, gid an int array of x's shape)."""
    out = np.zeros(n_groups, dtype=np.float32)
    np.maximum.at(out, gid.reshape(-1), np.abs(np.asarray(x, np.float32)).reshape(-1))
    return out


def group_ids(granularity: str, shape, row0: int = 0, col0: int = 0) -> tuple[np.ndarray, int]:
    """(group id of every element of a ``shape`` shard at (row0, col0), number of groups): blocks anchored at the
    global origin, rows, or matrices, numbered in row-major order."""
    *lead, n, k = shape
    m = int(np.prod(lead, dtype=np.int64))
    mat = np.arange(m).reshape(tuple(lead) + (1, 1)) if lead else np.zeros((1, 1), dtype=np.int64)
    if granularity == "tensor":
        return np.broadcast_to(mat, tuple(shape)).copy(), m
    if granularity == "channel":
        return (mat * n + np.arange(n)[:, None] + 0 * np.arange(k)[None, :]).astype(np.int64), m * n
    rows = (row0 + np.arange(n)) // 128 - row0 // 128
    cols = (col0 + np.arange(k)) // 128 - col0 // 128
    nr, nc = int(rows[-1]) + 1, int(cols[-1]) + 1
    return (mat * nr * nc + rows[:, None] * nc + cols[None, :]).astype(np.int64), m * nr * nc


def edge_amaxes_for(dtype: torch.dtype) -> np.ndarray:
    """edge_amaxes() restricted to the finite values ``dtype`` holds exactly, plus that dtype's own neighbours of
    448 * 2^k (one of its ulps above, and its largest value below 448 * 2^(k+1)) and its largest finite value."""
    if dtype == torch.float32:
        return edge_amaxes()
    top = float(torch.finfo(dtype).max)
    vals = [float(v) for v in edge_amaxes() if np.isfinite(v) and v <= top and float(torch.tensor(float(v)).to(dtype)) == float(v)]
    for k in (-20, -8, -1, 0, 1, 7, 40, 100):
        base = torch.tensor(448.0 * 2.0 ** k, dtype=dtype)
        if not torch.isfinite(base) or float(base) != 448.0 * 2.0 ** k:
            continue
        up = torch.nextafter(base, torch.tensor(float("inf"), dtype=dtype))
        down = torch.nextafter(2 * base, torch.tensor(0.0, dtype=dtype))
        vals += [float(v) for v in (up, down) if torch.isfinite(v)]
    vals.append(top)
    return np.unique(np.array(vals, dtype=np.float32))


def plant_edges(shape, dtype: torch.dtype, granularity: str, row0: int = 0, col0: int = 0, seed: int = 0):
    """A ``dtype`` shard whose groups (as ``group_ids``) take the amaxes edge_amaxes_for(dtype) in turn, then one
    all-zero (+-0) group and one all-subnormal group; later groups keep random finite data.  Each edge group holds
    its amax once (+-) among values of at most half of it.  -> (x, branch of every group)."""
    gid, n = group_ids(granularity, shape, row0, col0)
    vals = list(edge_amaxes_for(dtype))
    assert n >= len(vals) + 2, f"{n} groups for {len(vals) + 2} planted ones"
    u = synth_f32(tuple(shape), seed, spread=0).numpy()
    x = u * np.float32(4.0)
    tiny = np.float32(torch.finfo(dtype).tiny)
    first = {}
    for i, g in enumerate(gid.reshape(-1)):
        first.setdefault(int(g), i)
    flat, uf, gf = x.reshape(-1), u.reshape(-1), gid.reshape(-1)
    for j, v in enumerate(vals):
        sel = gf == j
        flat[sel] = uf[sel] * np.float32(0.5) * np.float32(v)
        flat[first[j]] = -v if j % 2 else v
    zero, sub = len(vals), len(vals) + 1
    flat[gf == zero] = np.where(uf[gf == zero] < 0, np.float32(-0.0), np.float32(0.0))
    flat[gf == sub] = uf[gf == sub] * tiny * np.float32(0.5)
    out = torch.from_numpy(x).to(dtype)
    amax = group_amax(widen(bits_of(out), str(dtype)[6:]), gid, n)
    return out, branch_of_amax(amax)


def plant_edge_sources(n_groups: int, group_shape, seed: int = 0) -> tuple[np.ndarray, np.ndarray]:
    """fp8 source groups whose dequantised amax takes every value of edge_amaxes() in turn (the byte 1.0 once under
    the scale v, the other bytes below 1.0), then an all-zero group and an all-subnormal one (scale 2^-140); later
    groups are random under scale 2^-3.  -> (q uint8 [n_groups, *group_shape], scale float32 [n_groups])."""
    vals = edge_amaxes()
    assert n_groups >= vals.size + 2
    rng = np.random.default_rng(seed)
    q = rng.integers(0, 0x38, size=(n_groups,) + tuple(group_shape), dtype=np.uint8) | \
        (rng.integers(0, 2, size=(n_groups,) + tuple(group_shape), dtype=np.uint8) << 7)
    s = np.full(n_groups, 2.0 ** -3, dtype=np.float32)
    first = (0,) * len(group_shape)
    for j, v in enumerate(vals):
        s[j] = v
        q[(j,) + first] = 0xB8 if j % 2 else 0x38  # -+1.0
    q[vals.size] = 0
    s[vals.size] = 1.0
    s[vals.size + 1] = np.float32(2.0 ** -140)
    return q, s


def pow2_scales(shape, seed: int, lo: int = -22, hi: int = 119) -> np.ndarray:
    """float32 powers of two 2^k, k uniform in [lo, hi] (both ends present when there are two entries or more)."""
    rng = np.random.default_rng(seed)
    k = rng.integers(lo, hi + 1, size=int(np.prod(shape, dtype=np.int64)))
    if k.size >= 2:
        k[0], k[-1] = lo, hi
    return np.ldexp(np.float32(1.0), k).astype(np.float32).reshape(shape)


def assert_pow2_over(s: torch.Tensor, s_f32: torch.Tensor) -> None:
    """Every finite UE8M0 scale_inv is a power of two, at least the float32 formula's scale_inv of the same group
    and below twice it; the non-finite ones sit where the float32 formula's do."""
    s, f = s.reshape(-1).float(), s_f32.reshape(-1).float()
    fin = torch.isfinite(s)
    assert torch.equal(fin, torch.isfinite(f)) and torch.equal(torch.isnan(s), torch.isnan(f))
    assert ((s[fin].view(torch.int32) & 0x7FFFFF) == 0).all()
    sd, fd = s[fin].double(), f[fin].double()
    assert (sd >= fd).all() and (sd < 2 * fd).all()

"""The fp8 casts (float8_e4m3fn, float8_e5m2) without a GPU: the C oracle against torch's recorded
bit patterns, the cast table of the C-ABI, the plan compiler's vector/scalar choice and kernel kind,
compiled fp8 plans replayed through the oracle, and how the Python layer names fp8 dtypes."""

import os
import random

import numpy as np
import pytest
import torch

from oracle import fp8_oracle
from tests.helpers import RectCase, rect_fields
from torchstore_b200 import _native
from torchstore_b200.direct_weight_sync import fused_refresh
from torchstore_b200.planner import StridedMem, build_rects, fill_rect

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "fp8_cast_vectors.npz")

E4M3, E5M2 = torch.float8_e4m3fn, torch.float8_e5m2
FP8 = (E4M3, E5M2)
WIDE = (torch.float32, torch.bfloat16, torch.float16)
FP8_PAIRS = [(s, d) for s in WIDE for d in FP8] + [(s, d) for s in FP8 for d in WIDE]
CODE = {torch.float32: _native.TSB_F32, torch.bfloat16: _native.TSB_BF16, torch.float16: _native.TSB_F16,
        torch.float64: _native.TSB_F64, E4M3: _native.TSB_F8E4M3, E5M2: _native.TSB_F8E5M2}
SHORT = {torch.float32: "f32", torch.bfloat16: "bf16", torch.float16: "f16", E4M3: "e4m3", E5M2: "e5m2"}
NP = {1: np.uint8, 2: np.uint16, 4: np.uint32}
# modes of csrc/tsb_internal.h: vector = MODE_<pair>_V16, scalar = vector + 1
VECTOR_MODE = {pair: 22 + 2 * i for i, pair in enumerate(
    [(torch.float32, E4M3), (torch.float32, E5M2), (torch.bfloat16, E4M3), (torch.bfloat16, E5M2),
     (torch.float16, E4M3), (torch.float16, E5M2), (E4M3, torch.float32), (E5M2, torch.float32),
     (E4M3, torch.bfloat16), (E5M2, torch.bfloat16), (E4M3, torch.float16), (E5M2, torch.float16)])}
KIND_GENERIC, KIND_B16, KIND_F32_BF16, KIND_BF16_E4M3 = 0, 1, 2, 3


@pytest.fixture(scope="module")
def vectors():
    return dict(np.load(GOLDEN))


def oracle_convert(bits: np.ndarray, src, dst) -> np.ndarray:
    bits = np.ascontiguousarray(bits)
    out = np.zeros(bits.size, dtype=NP[dst.itemsize])
    fp8_oracle.convert(bits.ctypes.data, CODE[src], out.ctypes.data, CODE[dst], bits.size, nan_mode=0)
    return out


def is_nan(bits: np.ndarray, dtype) -> np.ndarray:
    f = torch.from_numpy(bits.view({1: np.uint8, 2: np.int16, 4: np.int32}[dtype.itemsize]).copy())
    return torch.isnan(f.view(dtype).float()).numpy()


@pytest.mark.parametrize("src", ["f32", "bf16", "f16"])
@pytest.mark.parametrize("dst", [E4M3, E5M2])
def test_oracle_narrows_every_recorded_pattern_like_torch(vectors, src, dst):
    """Bit for bit, NaN encodings included: torch's fp8 narrowing keeps the sign of a NaN."""
    inp = vectors["f32"] if src == "f32" else vectors["all16"]
    sdt = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}[src]
    got = oracle_convert(inp, sdt, dst)
    want = vectors[f"{src}_to_{SHORT[dst]}"]
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, [(hex(int(inp[i])), hex(int(got[i])), hex(int(want[i]))) for i in bad[:8]]


@pytest.mark.parametrize("src", [E4M3, E5M2])
@pytest.mark.parametrize("dst", WIDE)
def test_oracle_widens_every_fp8_pattern_like_torch(vectors, src, dst):
    got = oracle_convert(vectors["all8"], src, dst)
    want = vectors[f"{SHORT[src]}_to_{SHORT[dst]}"]
    gn, wn = is_nan(got, dst), is_nan(want, dst)
    assert np.array_equal(gn, wn)
    assert np.array_equal(got[~wn], want[~wn])


@pytest.mark.parametrize("dst", [E4M3, E5M2])
def test_oracle_cuda_nan_mode_drops_the_sign_of_f16_nans(vectors, dst):
    """torch's CUDA .to() widens f16 with cvt.f32.f16, which makes every NaN positive: nan_mode=1
    (the CUDA encodings) differs from the CPU result exactly at the negative f16 NaNs."""
    bits = np.ascontiguousarray(vectors["all16"])
    out = np.zeros(bits.size, dtype=np.uint8)
    fp8_oracle.convert(bits.ctypes.data, CODE[torch.float16], out.ctypes.data, CODE[dst], bits.size, nan_mode=1)
    cpu = vectors[f"f16_to_{SHORT[dst]}"]
    neg_nan = ((bits & 0x7C00) == 0x7C00) & ((bits & 0x03FF) != 0) & ((bits & 0x8000) != 0)
    assert np.array_equal(out[~neg_nan], cpu[~neg_nan])
    assert (out[neg_nan] == 0x7F).all() and (cpu[neg_nan] == 0xFF).all()


def test_recorded_vectors_pin_the_saturation_rules(vectors):
    """The boundaries the kernel's fix-up of the .satfinite cvt depends on, read from torch's own output."""
    f32 = vectors["f32"]
    def at(value, key):
        i = np.nonzero(f32 == np.float32(value).view(np.uint32))[0][0]
        return int(vectors[key][i])
    assert at(448.0, "f32_to_e4m3") == 0x7E and at(464.0, "f32_to_e4m3") == 0x7E
    assert at(np.nextafter(np.float32(464.0), np.float32(1e9)), "f32_to_e4m3") == 0x7F
    assert at(-480.0, "f32_to_e4m3") == 0xFF and at(np.inf, "f32_to_e4m3") == 0x7F
    assert at(57344.0, "f32_to_e5m2") == 0x7B and at(61440.0, "f32_to_e5m2") == 0x7C
    assert at(np.nextafter(np.float32(61440.0), np.float32(0)), "f32_to_e5m2") == 0x7B
    assert at(-np.inf, "f32_to_e5m2") == 0xFC
    assert at(2.0 ** -10, "f32_to_e4m3") == 0x00 and at(np.nextafter(np.float32(2.0 ** -10), np.float32(1)), "f32_to_e4m3") == 0x01
    neg_nan = np.nonzero(f32 == np.uint32(0xFFC00000))[0][0]
    assert vectors["f32_to_e4m3"][neg_nan] == 0xFF and vectors["f32_to_e5m2"][neg_nan] == 0xFF


def test_cast_table_gains_exactly_the_twelve_fp8_pairs():
    codes = list(range(10))
    table = {(s, d): _native.lib().tsb_cast_supported(s, d) for s in codes for d in codes}
    fp8 = {(CODE[s], CODE[d]) for s, d in FP8_PAIRS}
    old = {(s, d) for s in range(8) for d in range(8) if s != d and table[(s, d)]}
    assert old == {(6, 5), (6, 4), (5, 6), (4, 6), (5, 4), (4, 5), (7, 6), (6, 7)}
    new = {(s, d) for (s, d), ok in table.items() if ok and s != d and (s >= 8 or d >= 8)}
    assert new == fp8
    assert all(table[(c, c)] for c in codes)
    assert not _native.lib().tsb_cast_supported(10, 10) and not _native.lib().tsb_cast_supported(8, 10)
    for s, d in FP8_PAIRS:
        assert _native.cast_supported(s, d)
    assert not _native.cast_supported(E4M3, E5M2) and not _native.cast_supported(torch.float64, E4M3)
    assert not _native.cast_supported(torch.int64, E4M3)


def test_same_dtype_fp8_stays_an_opaque_byte_move():
    assert _native.dtype_code(E4M3) == _native.dtype_code(E5M2) == _native.TSB_U8
    rect = _native.make_rect_array(1)[0]
    a = StridedMem(1 << 20, (64,), (1,), E4M3, 0)
    assert fill_rect(rect, a, StridedMem(2 << 20, (64,), (1,), E4M3, 0))
    assert rect.src_dtype == rect.dst_dtype == _native.TSB_U8
    assert fill_rect(rect, StridedMem(1 << 20, (64,), (1,), torch.bfloat16, 0), StridedMem(2 << 20, (64,), (1,), E4M3, 0))
    assert (rect.src_dtype, rect.dst_dtype) == (_native.TSB_BF16, _native.TSB_F8E4M3)
    assert fill_rect(rect, StridedMem(1 << 20, (64,), (1,), E5M2, 0), StridedMem(2 << 20, (64,), (1,), torch.float32, 0))
    assert (rect.src_dtype, rect.dst_dtype) == (_native.TSB_F8E5M2, _native.TSB_F32)
    with pytest.raises(NotImplementedError):
        fill_rect(rect, a, StridedMem(2 << 20, (64,), (1,), E5M2, 0))
    # the host tier moves bytes only
    r = _native.make_rect_array(1)
    fill_rect(r[0], StridedMem(1 << 20, (64,), (1,), torch.bfloat16, -1), StridedMem(2 << 20, (64,), (1,), E4M3, -1))
    with pytest.raises(_native.TsbError, match="host tier moves bytes"):
        _native.host_copy_rects(r, 1)


def compile_one(src: StridedMem, dst: StridedMem):
    rects, n = build_rects([(src, dst)])
    table, tiles, info = _native.plan_compile_host(0, rects, n)
    return rect_fields(table), info


BASE = 1 << 32


@pytest.mark.parametrize("pair", FP8_PAIRS, ids=lambda p: f"{SHORT[p[0]]}-{SHORT[p[1]]}")
def test_vector_mode_needs_16_byte_alignment_and_whole_16_element_runs(pair):
    s, d = pair
    vmode = VECTOR_MODE[pair]
    def mode(run, soff=0, doff=0, rows=1, spitch=None, dpitch=None):
        spitch = spitch or run
        dpitch = dpitch or run
        f, info = compile_one(StridedMem(BASE + soff * s.itemsize, (rows, run), (spitch, 1), s, 0),
                              StridedMem(BASE + (1 << 30) + doff * d.itemsize, (rows, run), (dpitch, 1), d, 0))
        assert len(f) == 1
        assert info.num_vector_rects == (1 if int(f["mode"][0]) == vmode else 0)
        return int(f["mode"][0]), f
    m, f = mode(64)
    assert m == vmode and int(f["units_per_row"][0]) == 4
    assert int(f["src_unit_bytes"][0]) == 16 * s.itemsize and int(f["dst_unit_bytes"][0]) == 16 * d.itemsize
    assert mode(16)[0] == vmode
    assert mode(24)[0] == vmode + 1                      # run not a multiple of 16 elements
    assert mode(8)[0] == vmode + 1                       # 8 elements: a vector unit of the 16-bit casts, not of fp8
    assert mode(64, soff=16)[0] == vmode                 # still 16-byte aligned on both sides
    assert mode(64, soff=1)[0] == vmode + 1              # source off alignment
    assert mode(64, doff=1)[0] == vmode + 1              # destination off alignment
    assert mode(32, rows=3, spitch=48, dpitch=48)[0] == vmode            # strided rows, 16-byte pitches
    assert mode(32, rows=3, spitch=40, dpitch=48)[0] == (vmode if 40 * s.itemsize % 16 == 0 else vmode + 1)
    m, f = mode(17)
    assert m == vmode + 1 and int(f["src_unit_bytes"][0]) == s.itemsize and int(f["dst_unit_bytes"][0]) == d.itemsize


def test_bf16_to_e4m3_kind_only_for_all_vector_bf16_e4m3_plans():
    def kind(pairs):
        rects, n = build_rects(pairs)
        return rect_fields(_native.plan_compile_host(0, rects, n)[0])
    def K(fields):  # Compiler::kind
        m = fields["mode"]
        if (m == 4).all():
            return KIND_B16
        if (m == 8).all():
            return KIND_F32_BF16
        if (m == VECTOR_MODE[(torch.bfloat16, E4M3)]).all():
            return KIND_BF16_E4M3
        return KIND_GENERIC
    bf = lambda off, n=256: StridedMem(BASE + off, (n,), (1,), torch.bfloat16, 0)
    f8 = lambda off, n=256, dt=E4M3: StridedMem(BASE + (1 << 30) + off, (n,), (1,), dt, 0)
    assert K(kind([(bf(0), f8(0)), (bf(4096), f8(4096))])) == KIND_BF16_E4M3
    assert K(kind([(bf(0), f8(0)), (bf(4096, 24), f8(4096, 24))])) == KIND_GENERIC        # one scalar rect
    assert K(kind([(bf(0), f8(0)), (bf(4096), f8(4096, dt=E5M2))])) == KIND_GENERIC       # e5m2
    assert K(kind([(bf(0), f8(0)), (bf(4096), bf(1 << 20))])) == KIND_GENERIC           # a byte move
    assert K(kind([(StridedMem(BASE, (256,), (1,), torch.float32, 0), f8(0))])) == KIND_GENERIC
    assert set(kind([(bf(0), f8(0))])["mode"].tolist()) == {VECTOR_MODE[(torch.bfloat16, E4M3)]}


# ---- compiled fp8 plans replayed through the oracle --------------------------------------------------
def fp8_case(rng: random.Random, edge: bool) -> RectCase:
    s, d = rng.choice(FP8_PAIRS)
    ndim = rng.choice([1, 2, 2, 3])
    if edge:  # around the vector rule: runs of 16k +- 1 elements, 16-byte aligned or one element off
        shape = [rng.choice([1, 2, 3, 7]) for _ in range(ndim - 1)] + [16 * rng.randint(1, 40) + rng.choice([-1, 0, 0, 1])]
    else:
        shape = [rng.choice([1, 2, 3, 5, 8, 16, 17, 31, 32, 64, 100, 257]) for _ in range(ndim)]
    def window(dtype):
        q = max(1, 16 // dtype.itemsize)
        start = q * rng.randint(0, 2) if rng.random() < 0.6 else rng.randint(1, 3)
        inner = -(-(start + shape[-1]) // q) * q + q * rng.randint(0, 2)
        base = [e + rng.choice([0, 1]) for e in shape[:-1]] + [inner]
        starts = [rng.randint(0, b - e) for b, e in zip(base[:-1], shape[:-1])] + [start]
        return tuple(base), tuple(slice(a, a + e) for a, e in zip(starts, shape))
    (sb, si), (db, di) = window(s), window(d)
    return RectCase(sb, db, s, d, lambda b, i=si: b[i], lambda b, i=di: b[i])


def host_bases(cases, seed):
    gen = torch.Generator().manual_seed(seed)
    out = []
    for c in cases:
        n = int(np.prod(c.src_base_shape))
        src = torch.randint(0, 256, (n * c.src_dtype.itemsize,), dtype=torch.uint8, generator=gen).view(c.src_dtype)
        src = src.reshape(c.src_base_shape)
        dst = torch.full((int(np.prod(c.dst_base_shape)) * c.dst_dtype.itemsize,), 0x33, dtype=torch.uint8)
        dst = dst.view(c.dst_dtype).reshape(c.dst_base_shape)
        out.append((c.src_view(src), c.dst_view(dst), dst, src))
    return out


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
@pytest.mark.parametrize("tile_units", [0, 64])
def test_compiled_fp8_plans_replay_to_the_oracle(seed, tile_units):
    rng = random.Random(4242 + seed)
    cases = [fp8_case(rng, edge=i % 2 == 1) for i in range(40)]
    direct = host_bases(cases, seed)
    replay = host_bases(cases, seed)
    rects, n = build_rects([(StridedMem.from_tensor(p[0]), StridedMem.from_tensor(p[1])) for p in direct])
    fp8_oracle.copy_rects(rects, n, nan_mode=1)
    rects2, n2 = build_rects([(StridedMem.from_tensor(p[0]), StridedMem.from_tensor(p[1])) for p in replay])
    table, tiles, info = _native.plan_compile_host(0, rects2, n2, 0, tile_units)
    modes = set(rect_fields(table)["mode"].tolist())
    assert modes <= set(range(22, 46))
    assert any(m % 2 == 0 for m in modes) and any(m % 2 == 1 for m in modes)
    fp8_oracle.replay_plan(table, tiles, tile_units or info.tile_bytes // 16, nan_mode=1)
    for (_, _, want, _), (_, _, got, _) in zip(direct, replay):
        assert torch.equal(got.view(torch.uint8), want.view(torch.uint8))


def test_refresh_route_fuses_exactly_the_kernel_pairs():
    """register(transfer_dtype=...): params with a fused cast go to the batched refresh plan, every
    other one (int buffers, float64 staging, fp8 -> fp8 of another format) to staging.copy_."""
    for s, d in FP8_PAIRS:
        assert fused_refresh(s, d)
    assert fused_refresh(torch.float32, torch.bfloat16) and fused_refresh(E4M3, E4M3)
    assert fused_refresh(torch.int64, torch.int64)
    for s, d in [(torch.int64, E4M3), (torch.float64, E4M3), (torch.float32, torch.int32),
                 (torch.bfloat16, torch.float64), (E4M3, E5M2), (torch.int32, torch.bfloat16)]:
        assert not fused_refresh(s, d), (s, d)

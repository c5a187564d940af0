"""The scaled-fp8 kernels on the H100 in every regime of tests/fp8_regimes.py, past byte 2^32 of their
allocations, and across random layouts of all four scaled plan kinds.

* Regimes: every catalogue workload pulled through DirectWeightSyncDest.pull with finite data, with a poisoned
  source scale (Inf, NaN, 0 and a negative scale) and with an all-zero destination group; the regime asserted
  again from the tables of the live plan's inputs (and their size against plan_info); bit-exact against the
  numpy oracle wherever it is not NaN, against the torch CUDA composition with NaN bytes included; guard bytes
  around the weight and the scale tensor.  The dequantising regimes also run from int8 handles (``src_dtype``: the
  bytes of ``int8_of``, checked against oracle/int8_source_oracle.py and its torch rendering).
* Past 32 bits: a requantising and a dequantising pull of a fp8 MoE stack whose source shard and destination
  both extend past byte 2^32.
* Random layouts: seeded draws of a global shape, a source layout (FSDP rows starting mid-block, column
  shards, replicas, EP), a source granularity or dtype and a destination window, for quantising, dequantising
  and requantising pulls; mixed seeds put all five plan kinds (plain, cast, quantise, dequantise, requantise)
  in one pull and replay it."""

import asyncio
import contextlib
import random

import numpy as np
import pytest
import torch

from oracle import block_fp8_oracle, int8_source_oracle, scaled_fp8_oracle
from oracle.dequant_fp8_oracle import DST, GRANULARITIES, torch_dequantize
from oracle.requant_fp8_oracle import SCALE_POISON, torch_requantize
from tests import test_gpu_dequant_fp8 as dq_gpu
from tests import test_gpu_requant_fp8 as rq_gpu
from tests.fp8_regimes import REGIMES, WORKLOADS, Workload, geometry, split, whole
from tests.helpers import region, shard_box
from tests.test_gpu_dequant_fp8 import KW, cleanup, guarded, guards_intact, register
from tests.test_requant_fp8_cpu import CODE, dest_scale_shape, fp8_full, global_scale, local_scale
from torchstore_b200 import _native
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource, _add_dq_source
from torchstore_b200.planner import build_rects
from torchstore_b200.transport.types import TensorSlice

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
E4M3 = torch.float8_e4m3fn
POISON = (float(SCALE_POISON[0]), float(SCALE_POISON[1]), 0.0, -0.5)  # Inf, NaN, 0, negative


@pytest.fixture(scope="module", autouse=True)
def _init():
    _native.init()
    yield


def run(coro):
    return asyncio.run(coro)


@contextlib.contextmanager
def named(what):
    """Prefix a failing comparison with the layout it ran on."""
    try:
        yield
    except AssertionError as e:
        raise AssertionError(f"{what}: {e}") from e


# ---- the live plan's tables -------------------------------------------------------------------------
def live_tables(sync, dest, dest_scale=None, dg=None, int8_src=False):
    """Compile on the host the tables of the plan `sync` built for its one name: the same windows, sources and
    target it compiled from, with the live device addresses (`int8_src`: a dequantising plan of int8 handles, TSB_I8
    rects).  Checks their size against plan_info and returns (tables, Geometry)."""
    dev = dest.device.index
    pairs, sources = [], {}
    for op in sync._plan:
        pairs.append(DirectWeightSyncDest.op_windows(op, op.rdma_buffer.window(dev)))
        _add_dq_source(sources, op, dev)
    arr = _native.make_dq_source_array(max(1, len(sources)))
    for i, (_, s) in enumerate(sources.values()):
        arr[i] = s
    rects, n = build_rects(pairs, dequantise=int8_src)
    *lead, rows, cols = dest.shape
    if dg is None:
        tables = _native.dequant_fp8_compile_host(dev, rects, n, arr, len(sources))
        mine, other = (sync._int8_dequant_plans, sync._dequant_plans) if int8_src else (sync._dequant_plans, sync._int8_dequant_plans)
        assert not other, "dequantising plans of the other source format"
        info = _native.plan_info(mine[dev])
        count, read = len(tables), int((tables["rows"].astype(np.int64) * tables["cols"]).sum())
    else:
        for i in range(n):
            rects[i].src_dtype = rects[i].dst_dtype = _native.TSB_F8E4M3
        tgt = _native.make_sq_target_array(1)
        tgt[0] = _native.SqTarget(dest.data_ptr(), dest_scale.data_ptr(), dest.numel() // (rows * cols), rows, cols, CODE[dg], 0)
        tables = _native.requant_fp8_compile_host(dev, rects, n, arr, len(sources), tgt, 1)
        units, pieces, tiles, _ = tables
        info = _native.plan_info(sync._requant_plans[dev])
        count = len(units) + len(tiles)
        read = int((pieces["rows"].astype(np.int64) * pieces["cols"]).sum() + (tiles["rows"].astype(np.int64) * tiles["cols"]).sum())
    assert (info.num_tiles, info.src_bytes) == (count, read)
    return tables, geometry(dest.data_ptr(), tuple(dest.shape), dest.element_size(), arr, len(sources))


# ---- the regimes ------------------------------------------------------------------------------------
def poison(s, seed):
    """Inf, NaN, 0 and -0.5 at four spread entries of a source scale (one of them if it has one entry)."""
    flat = s.reshape(-1)
    n = flat.numel()
    for k, i in enumerate(sorted({0, n // 3, 2 * n // 3, n - 1})):
        flat[i] = POISON[(k + seed) % len(POISON)]
    return s


def zero_first_group(q, w: Workload):
    """All-zero bytes over the first destination group of `w` (dequantising pulls: its first row)."""
    off, loc = w.dst
    *lead, n, k = loc
    h, kk = {"block": (min(128, n), min(128, k)), "channel": (1, k), "tensor": (n, k)}.get(w.out, (1, k))
    q.view(torch.uint8)[tuple(off[:-2]) + (slice(off[-2], off[-2] + h), slice(off[-1], off[-1] + kk))] = 0
    return q


def inputs(w: Workload, variant: str, src_dtype=E4M3):
    """The source weight (fp8 bytes, or int8 ones from int8_of) and its global scale of workload `w` in `variant`."""
    q = int8_source_oracle.int8_of(w.shape, w.seed) if src_dtype == torch.int8 else fp8_full(w.shape, w.seed)
    s = global_scale(w.sg, w.shape, w.seed)
    if variant == "poisoned_scale":
        s = poison(s, w.seed)
    elif variant == "zero_group":
        q = zero_first_group(q, w)
    return q, s


VARIANTS = ("finite", "poisoned_scale", "zero_group")


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("regime", sorted(REGIMES))
def test_regime_on_the_h100(regime, variant):
    run_regime(regime, variant)


def run_regime(regime, variant, scale_fmt=None, src_dtype=E4M3):
    """Pull the regime's workload in `variant` (requantising ones with the scale format `scale_fmt`; dequantising
    ones from handles of `src_dtype`, float8_e4m3fn or int8) and check it."""
    r = REGIMES[regime]
    w = WORKLOADS[r.workload]
    int8 = src_dtype == torch.int8
    assert not (int8 and w.kind == "requant"), "int8 handles are not requantised"
    q, s = inputs(w, variant, src_dtype)
    sources, handles = register(q, s, w.sg, list(w.src))
    where = f"{regime} ({r.doc}), {variant}, scale_fmt={scale_fmt}, {src_dtype}: {w.describe()}"
    if w.kind == "requant":
        sync, y, ys, bases = rq_gpu.pull_into(handles, w.shape, w.dst, w.out, scale_fmt=scale_fmt)
        tables, geom = live_tables(sync, y, ys, w.out)
        assert r.holds(tables, geom), f"not reached: {where}"
        with named(where):
            rq_gpu.assert_oracle(y, ys, q, s, w.sg, w.dst, w.out, scale_fmt)
            rq_gpu.assert_torch_cuda(y, ys, q, s, w.sg, w.dst, w.out, scale_fmt)
    else:
        sync, y, base = dq_gpu.pull_into(handles, w.shape, w.dst, DST[w.out])
        tables, geom = live_tables(sync, y, int8_src=int8)
        assert r.holds(tables, geom), f"not reached: {where}"
        with named(where):
            if int8:
                assert_int8_dequantised(y, q, s, w.sg, w.dst)
            else:
                dq_gpu.assert_oracle(y, dq_gpu.want_bits(q, s, w.sg, w.dst, DST[w.out]))
                dq_gpu.assert_torch_cuda(y, q, s, w.sg, w.dst)
        bases = (base,)
    assert all(guards_intact(b) for b in bases), where
    sync.close()
    cleanup(sources)


def assert_int8_dequantised(y, q, s, g, box):
    """A destination y dequantised from the `box` of int8 handles (q, global scale s): bit for bit the numpy oracle
    (NaN-agnostic) and the torch CUDA rendering (NaN bytes included)."""
    off, loc = box
    qr, sr = region(q, off, loc), local_scale(s, g, off, loc)
    dq_gpu.assert_oracle(y, int8_source_oracle.dequantize(qr.numpy(), sr.numpy(), g, off[-2], off[-1], str(y.dtype)[6:]))
    want = int8_source_oracle.torch_dequantize(qr.to(DEV), sr.to(DEV), g, off[-2], off[-1], y.dtype)
    assert torch.equal(y.view(torch.uint8), want.view(torch.uint8))


# ---- past byte 2^32 ---------------------------------------------------------------------------------
def big_stack(experts, rows, cols, seed):
    """A finite fp8 MoE stack on the GPU, one expert at a time (no full-size temporary)."""
    gen = torch.Generator(DEV).manual_seed(seed)
    q = torch.empty(experts, rows, cols, dtype=torch.uint8, device=DEV)
    for e in range(experts):
        b = torch.randint(0, 0x7F, (rows, cols), dtype=torch.uint8, device=DEV, generator=gen)  # 0x00..0x7E: finite
        q[e] = b | (torch.randint(0, 2, (rows, cols), dtype=torch.uint8, device=DEV, generator=gen) << 7)
    return q.view(E4M3)


def skip_unless_free(nbytes):
    free, _ = torch.cuda.mem_get_info(DEV)
    if free < 3 * nbytes:
        pytest.skip(f"needs {3 * nbytes / 2**30:.1f} GiB of free device memory, {free / 2**30:.1f} GiB free")


def test_requantise_past_byte_2_32():
    """A block-scaled fp8 stack of 129 experts [4096, 8192] (4.3 GB) into a per-channel destination: the source
    shard and the destination both run past byte 2^32; the last matrices against the torch CUDA composition."""
    shape = (129, 4096, 8192)
    n = int(np.prod(shape))
    assert n > 2**32
    skip_unless_free(2 * n)
    q = big_stack(*shape, seed=1)
    s = global_scale("block", shape, 1).to(DEV)
    sources, handles = register(q, s, "block", [whole(shape)])
    sync, y, ys, bases = rq_gpu.pull_into(handles, shape, whole(shape), "channel")
    for e in (0, shape[0] - 2, shape[0] - 1):
        want_q, want_s = torch_requantize(q[e], s[e], "block", 0, 0, "channel")
        assert torch.equal(y[e].view(torch.uint8), want_q.view(torch.uint8)), e
        assert torch.equal(ys[e].view(torch.int32), want_s.view(torch.int32)), e
    assert all(guards_intact(b) for b in bases)
    sync.close()
    cleanup(sources)
    del q, y, ys, bases, sources, handles
    torch.cuda.empty_cache()


def test_dequantise_past_byte_2_32():
    """A channel-scaled fp8 stack of 129 experts [4096, 8192] (4.3 GB) into bf16 (8.7 GB): the source shard and
    the destination both run past byte 2^32; the last matrices against the torch CUDA rendering."""
    shape = (129, 4096, 8192)
    n = int(np.prod(shape))
    skip_unless_free(3 * n)
    q = big_stack(*shape, seed=2)
    s = global_scale("channel", shape, 2).to(DEV)
    sources, handles = register(q, s, "channel", [whole(shape)])
    sync, y, base = dq_gpu.pull_into(handles, shape, whole(shape), torch.bfloat16)
    for e in (0, shape[0] - 2, shape[0] - 1):
        assert torch.equal(y[e], torch_dequantize(q[e], s[e], "channel")), e
    assert guards_intact(base)
    sync.close()
    cleanup(sources)
    del q, y, base, sources, handles
    torch.cuda.empty_cache()


# ---- random layouts across the four scaled plan kinds ----------------------------------------------
WIDTHS = (16, 48, 64, 100, 128, 130, 260, 16384, 16400, 32768, 32784)
SRC_DTYPES = (torch.bfloat16, torch.float16, torch.float32)


def draw(rng: random.Random, kind: str, seed: int) -> Workload:
    """One random pull of `kind` ("quant", "dequant" or "requant")."""
    k = rng.choice(WIDTHS)
    n = rng.randint(1, max(1, min(400, 300_000 // k)))
    shape = (rng.randint(2, 4), n, k) if rng.random() < 0.3 else (n, k)
    layout = rng.choice(["rows", "cols", "replica"] + (["ep"] * (len(shape) == 3)))
    if layout == "rows":
        src = split(shape, rng.randint(2, 6), -2)
    elif layout == "cols":
        src = split(shape, rng.randint(2, 4), -1)
    elif layout == "replica":
        src = split(shape, 2, -2) * 2
    else:
        src = split(shape, shape[0], 0)
    src = tuple(b for b in src if 0 not in b[1])
    tp = rng.choice(["whole", "rows", "cols"])
    dst = whole(shape) if tp == "whole" else shard_box(shape, 2, rng.randint(0, 1), len(shape) - (2 if tp == "rows" else 1))
    if 0 in dst[1]:
        dst = whole(shape)
    sg = rng.choice(SRC_DTYPES) if kind == "quant" else rng.choice(GRANULARITIES)
    out = rng.choice(list(DST)) if kind == "dequant" else rng.choice(GRANULARITIES)
    return Workload(kind, shape, str(sg).replace("torch.", ""), src, dst, out, seed)


class Case:
    """One name of a pull drawn by draw(): its sources, its destination and its check."""

    def __init__(self, name: str, w: Workload):
        self.name, self.w = name, w
        self.scale = self.y_scale = None
        if w.kind == "quant":
            self.x = (torch.randn(w.shape, generator=torch.Generator().manual_seed(w.seed)) * 0.05).to(getattr(torch, w.sg))
            self.sources = []
            self.handles = []
            for r, (off, loc) in enumerate(w.src):
                src = DirectWeightSyncSource()
                sl = TensorSlice(off, (r,), w.shape, loc, (len(w.src),))
                self.handles.append(src.register({name: region(self.x, off, loc).contiguous().to(DEV)}, rank=r,
                                                 tensor_slices={name: sl})[name])
                self.sources.append((src,))
        else:
            self.q, self.scale = fp8_full(w.shape, w.seed), global_scale(w.sg, w.shape, w.seed)
            self.sources, self.handles = register(self.q, self.scale, w.sg, list(w.src), name=name)
        loc = w.dst[1]
        if w.kind == "dequant":
            self.base, self.y = guarded(loc, DST[w.out])
            self.bases = (self.base,)
        else:
            qb, self.y = guarded(loc, E4M3)
            sb, self.y_scale = guarded(dest_scale_shape(w.out, loc), torch.float32)
            self.bases = (qb, sb)

    def slice(self):
        off, loc = self.w.dst
        return TensorSlice(off, (0,), self.w.shape, loc, (1,))

    def check(self):
        w, (off, loc) = self.w, self.w.dst
        if w.kind == "quant":
            x = region(self.x, off, loc).float().numpy()
            want_q, want_s = block_fp8_oracle.quantize(x) if w.out == "block" else scaled_fp8_oracle.quantize(x, w.out)
            assert np.array_equal(self.y.view(torch.uint8).cpu().numpy(), want_q)
            assert np.array_equal(self.y_scale.cpu().numpy().reshape(-1).view(np.uint32), np.asarray(want_s, np.float32).reshape(-1).view(np.uint32))
        elif w.kind == "dequant":
            dq_gpu.assert_oracle(self.y, dq_gpu.want_bits(self.q, self.scale, w.sg, w.dst, DST[w.out]))
            dq_gpu.assert_torch_cuda(self.y, self.q, self.scale, w.sg, w.dst)
        else:
            rq_gpu.assert_oracle(self.y, self.y_scale, self.q, self.scale, w.sg, w.dst, w.out)
            rq_gpu.assert_torch_cuda(self.y, self.y_scale, self.q, self.scale, w.sg, w.dst, w.out)
        assert all(guards_intact(b) for b in self.bases)

    def close(self):
        cleanup(self.sources)


def pull_cases(sync, cases, extra_handles=None, extra_dest=None):
    handles = {c.name: c.handles for c in cases}
    dest = {c.name: c.y for c in cases}
    slices = {c.name: c.slice() for c in cases}
    scales = {kw: {} for kw in KW.values()}
    for c in cases:
        if c.y_scale is not None:
            scales[KW[c.w.out]][c.name] = c.y_scale
    handles.update(extra_handles or {})
    dest.update(extra_dest or {})
    run(sync.pull(handles, dest, slices, **{k: v for k, v in scales.items() if v}, requantize=True))


@pytest.mark.parametrize("seed", range(48))
def test_random_layouts_match_the_oracles(seed):
    rng = random.Random(9000 + seed)
    kind = ("quant", "dequant", "requant")[seed % 3]
    w = draw(rng, kind, seed)
    case = Case("w", w)
    sync = DirectWeightSyncDest()
    try:
        with named(f"seed {seed}: {w.describe()}"):
            pull_cases(sync, [case])
            case.check()
    finally:
        sync.close()
        case.close()


@pytest.mark.parametrize("seed", range(6))
def test_random_mixed_pull_of_all_five_kinds_replays(seed):
    """One pull with a plain copy, a fused cast and random quantising, dequantising and requantising names;
    the replay (destinations overwritten first) lands the same bytes."""
    rng = random.Random(9500 + seed)
    cases = [Case(kind, draw(rng, kind, 100 * seed + i)) for i, kind in enumerate(("quant", "dequant", "requant"))]
    plain = (torch.randn(96, 80) * 0.1).to(torch.bfloat16)
    cast = torch.randn(64, 48)
    src = DirectWeightSyncSource()
    h = src.register({"plain": plain.to(DEV), "cast": cast.to(DEV)}, rank=0)
    dest = {"plain": torch.zeros(96, 80, dtype=torch.bfloat16, device=DEV), "cast": torch.zeros(64, 48, dtype=torch.bfloat16, device=DEV)}
    sync = DirectWeightSyncDest()
    layouts = "; ".join(f"{c.name}: {c.w.describe()}" for c in cases)
    try:
        with named(f"seed {seed}: {layouts}"):
            pull_cases(sync, cases, {"plain": [h["plain"]], "cast": [h["cast"]]}, dest)
            assert sync._native_plans and sync._dequant_plans and sync._requant_plans
            assert sync._block_plans or sync._scaled_plans
            for c in cases:
                c.check()
            assert torch.equal(dest["plain"].cpu(), plain) and torch.equal(dest["cast"], cast.to(DEV).to(torch.bfloat16))
            first = [t.clone() for c in cases for t in (c.y, c.y_scale) if t is not None] + [dest["plain"].clone(), dest["cast"].clone()]
            for c in cases:
                c.y.view(torch.uint8).fill_(0xA5)
                if c.y_scale is not None:
                    c.y_scale.fill_(-3.0)
            dest["plain"].zero_()
            dest["cast"].zero_()
            before = dict(sync._requant_plans)
            pull_cases(sync, cases, {"plain": [h["plain"]], "cast": [h["cast"]]}, dest)
            assert dict(sync._requant_plans) == before  # replayed, not rebuilt
            again = [t for c in cases for t in (c.y, c.y_scale) if t is not None] + [dest["plain"], dest["cast"]]
            assert all(torch.equal(a.reshape(-1).view(torch.uint8), b.reshape(-1).view(torch.uint8)) for a, b in zip(first, again))
    finally:
        sync.close()
        for c in cases:
            c.close()
        run(src.cleanup())

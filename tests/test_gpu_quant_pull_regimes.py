"""The quantising pulls on the H100 in every regime of tests/quant_pull_regimes.py, in a mixed-dtype dict, past
byte 2^32 of their allocations, and across random layouts with special values.

* Regimes: every catalogue workload pulled through DirectWeightSyncDest.pull with block_scales / channel_scales
  / tensor_scales, with finite data; with NaN, +-Inf, all-zero and subnormal groups, -0 and subnormal values at
  the places the kernels branch (warp steps that span rows, the ends of byte-wise pieces, pieces off a 16-byte
  column, partial block corners); with values at the top of the source dtype; and after an in-place update of
  every source shard, pulled again over guard-filled destinations by the same plans.  The regime is asserted
  again from the tables of the live plan's inputs (and their size against plan_info); weights and scale_inv
  are compared bit for bit with the numpy oracle (NaN-agnostic inside non-finite groups) and with the torch
  CUDA composition (NaN bytes included), and the guard bytes around both are checked.
* A mixed dict: bf16, f16 and f32 names at every granularity beside a plain and a cast name in one pull,
  replayed over overwritten destinations.
* Past 32 bits: a bf16 MoE stack whose source runs past byte 2^32 and whose fp8 destination does too.
* Random layouts: seeded draws of a global shape, source shards and a destination window with NaN, Inf,
  zero and subnormal groups planted at shard, block and row boundaries.

The regime and random-layout runners take the destination dtype (``dst_dtype``, float8_e4m3fn by default; int8
destinations are checked against oracle/int8_oracle.py and its torch rendering)."""

import asyncio
import random

import numpy as np
import pytest
import torch

from oracle import block_fp8_oracle, int8_source_oracle, scaled_fp8_oracle, ue8m0_oracle
from oracle.block_fp8_oracle import synth_f32
from tests import test_gpu_block_fp8 as bq_gpu
from tests.fp8_regimes import split, whole
from tests.helpers import rand_full, region
from tests import test_gpu_scaled_fp8 as sq_gpu
from tests.quant_pull_regimes import (BLOCK, ES, GRANULARITIES, KW, REGIMES, WORKLOADS, Pull, compile_tables, plan_bytes,
                                      scale_shape, spots)
from tests.test_block_fp8_cpu import assert_block_fp8_equal
from tests.test_gpu_dequant_fp8 import guarded, guards_intact
from tests.test_gpu_fp8_regimes import draw, named, skip_unless_free
from tests.test_gpu_source_quant_regimes import on_device
from tests.test_quant_pull_regimes_cpu import compiled, oracle_quantize, workload_inputs
from tests.test_scaled_fp8_cpu import assert_scaled_fp8_equal
from torchstore_b200 import _native
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource
from torchstore_b200.transport.types import TensorSlice

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
E4M3 = torch.float8_e4m3fn
TOP = {d: float(torch.finfo(getattr(torch, d)).max) for d in ES}  # 3.39e38, 65504, 3.40e38


@pytest.fixture(scope="module", autouse=True)
def _init():
    _native.init()
    yield


def run(coro):
    return asyncio.run(coro)


# ---- groups of a destination window -----------------------------------------------------------------
def group_of(p: Pull, coord) -> tuple:
    """The destination group (block, row or matrix of the window) holding global element `coord`."""
    *lead, r, c = (x - o for x, o in zip(coord, p.dst[0]))
    if p.g == "block":
        return (*lead, r // BLOCK, c // BLOCK)
    return (*lead, r) if p.g == "channel" else tuple(lead)


def group_box(p: Pull, key) -> tuple:
    """Global index of every element of destination group `key`."""
    (*lo, r0, c0), (*_, n, k) = p.dst
    lead = tuple(o + i for o, i in zip(lo, key))
    if p.g == "block":
        br, bc = key[-2:]
        return lead + (slice(r0 + br * BLOCK, r0 + min(n, (br + 1) * BLOCK)), slice(c0 + bc * BLOCK, c0 + min(k, (bc + 1) * BLOCK)))
    if p.g == "channel":
        return lead + (slice(r0 + key[-1], r0 + key[-1] + 1), slice(c0, c0 + k))
    return lead + (slice(r0, r0 + n), slice(c0, c0 + k))


def n_groups(p: Pull) -> int:
    *lead, n, k = p.dst[1]
    m = int(np.prod(lead, dtype=np.int64))
    return m * -(-n // BLOCK) * -(-k // BLOCK) if p.g == "block" else m * n if p.g == "channel" else m


def fill_group(x, p: Pull, key, kind: str, seed: int):
    box = group_box(p, key)
    shape = tuple(x[box].shape)
    if kind == "zero":
        x[box] = torch.where(synth_f32(shape, seed) < 0, -0.0, 0.0)
    else:
        x[box] = synth_f32(shape, seed, spread=0) * torch.finfo(getattr(torch, p.dtype)).tiny * 0.5


KINDS = ("nan", "inf", "-inf", "zero", "subnormal")


def plant_special(x, p: Pull, coords, seed: int):
    """NaN, +Inf, -Inf, an all-zero (+-0) group and an all-subnormal group, each in its own destination group
    at the first spots that lie in one (one group of the window keeps finite data when it has several); -0 and
    single subnormals at the spots in the other groups."""
    x = x.float().clone()
    kinds = {}
    for j, c in enumerate(coords):
        key = group_of(p, c)
        if key not in kinds and len(kinds) < max(1, n_groups(p) - 1):
            kinds[key] = KINDS[len(kinds) % len(KINDS)]
            if kinds[key] in ("zero", "subnormal"):
                fill_group(x, p, key, kinds[key], seed + j)
        kind = kinds.get(key)
        if kind in ("nan", "inf", "-inf"):
            x[c] = float(kind)
        elif kind is None:
            x[c] = -0.0 if j % 2 else torch.finfo(getattr(torch, p.dtype)).tiny * 0.25
    return x.to(getattr(torch, p.dtype))


def near_top(x, p: Pull, coords, seed: int):
    """Values of magnitude [0.25, 1] x the largest finite value of the source dtype, +-that value at the spots."""
    top = TOP[p.dtype]
    u = synth_f32(tuple(x.shape), seed, spread=0)
    y = u.sign() * (0.25 + 0.75 * u.abs()) * top
    for j, c in enumerate(coords):
        y[c] = top if j % 2 == 0 else -top
    return y.to(getattr(torch, p.dtype))


def inputs(name: str, variant: str):
    xs = workload_inputs(name)
    if variant not in ("special", "near_top"):
        return xs
    w = WORKLOADS[name]
    tables, geom, *_ = compiled(name)
    at = spots(tables, geom)
    plant = plant_special if variant == "special" else near_top
    return [plant(x, p, at.get(i, []), w.seed + 100 * i) for i, (p, x) in enumerate(zip(w.pulls, xs))]


# ---- one pull of several names ----------------------------------------------------------------------
class Pulled:
    """The names w0, w1, ... of `pulls` registered shard by shard (one source each), pulled into guarded
    destinations of `dst_dtype` (float8_e4m3fn or int8) and scales by one DirectWeightSyncDest with the scale format
    `scale_fmt`; `extra` handles and destinations join the pull."""

    def __init__(self, pulls, xs, extra_handles=None, extra_dests=None, scale_fmt=None, dst_dtype=E4M3):
        self.pulls, self.sources, self.shards, self.scale_fmt = tuple(pulls), [], {}, scale_fmt
        self.dst_dtype = dst_dtype
        self.handles, self.dests, self.scales, self.slices, self.bases = {}, {}, {}, {}, []
        try:
            for i, (p, x) in enumerate(zip(pulls, xs)):
                n = f"w{i}"
                self.handles[n], self.shards[n] = [], []
                for r, (off, loc) in enumerate(p.src):
                    shard = on_device(region(x, off, loc).contiguous(), p.shift(r))
                    src = DirectWeightSyncSource()
                    self.sources.append(src)
                    sl = TensorSlice(off, (r,), p.shape, loc, (len(p.src),))
                    self.handles[n].append(src.register({n: shard}, rank=r, tensor_slices={n: sl})[n])
                    self.shards[n].append(shard)
                qb, self.dests[n] = guarded(p.dst[1], dst_dtype)
                sb, self.scales[n] = guarded(scale_shape(p.g, p.dst[1]), torch.float32)
                self.bases += [qb, sb]
                self.slices[n] = TensorSlice(p.dst[0], (0,), p.shape, p.dst[1], (1,))
        except BaseException:
            self.close()
            raise
        self.all_handles = {**self.handles, **(extra_handles or {})}
        self.all_dests = {**self.dests, **(extra_dests or {})}
        self.by_kw = {}
        for i, p in enumerate(self.pulls):
            self.by_kw.setdefault(KW[p.g], {})[f"w{i}"] = self.scales[f"w{i}"]
        self.sync = DirectWeightSyncDest()

    def pull(self):
        run(self.sync.pull(self.all_handles, self.all_dests, self.slices, **self.by_kw, scale_fmt=self.scale_fmt))

    def plan_dicts(self):
        """The (block, per-channel / per-tensor) plans of the destination format; the other format's stay empty."""
        fp8, int8 = (self.sync._block_plans, self.sync._scaled_plans), (self.sync._int8_block_plans, self.sync._int8_scaled_plans)
        mine, other = (int8, fp8) if self.dst_dtype == torch.int8 else (fp8, int8)
        assert not any(other), "plans of the other destination format"
        return mine

    def plans(self):
        return tuple(dict(p) for p in self.plan_dicts())

    def live_tables(self):
        """The tables of the plans the pull built, compiled on the host from the same windows and targets with
        the live device addresses; their size checked against plan_info."""
        tables, geom = compile_tables(self.pulls, self.sync._plan, self.handles, lambda b: b.window(0), self.dests, self.scales)
        want = plan_bytes(tables)
        for kind, plans in zip(("block", "scaled"), self.plan_dicts()):
            if kind in want:
                info = _native.plan_info(plans[0])
                assert (info.num_tiles, info.src_bytes) == want[kind], kind
            else:
                assert not plans, kind
        return tables, geom

    def check(self, xs):
        for i, (p, x) in enumerate(zip(self.pulls, xs)):
            n = f"w{i}"
            with named(f"w{i}: {p.describe()}"):
                assert_quantised(self.dests[n], self.scales[n], region(x, *p.dst), p.g, self.scale_fmt, self.dst_dtype)
        assert all(guards_intact(b) for b in self.bases)

    def update(self, xs):
        """New values in every source shard, in place; guard patterns over every destination and scale."""
        for i, (p, x) in enumerate(zip(self.pulls, xs)):
            for shard, (off, loc) in zip(self.shards[f"w{i}"], p.src):
                shard.copy_(region(x, off, loc).to(DEV))
            self.dests[f"w{i}"].view(torch.uint8).fill_(0xA5)
            self.scales[f"w{i}"].fill_(-3.0)

    def close(self):
        if hasattr(self, "sync"):
            self.sync.close()
        for src in self.sources:
            run(src.cleanup())


def assert_quantised(y, ys, x, g, scale_fmt=None, dst_dtype=E4M3):
    """The fp8 weight y and its scale_inv ys against the numpy oracle of the source region x (bit-exact in
    finite groups, NaN-agnostic in the others) and the torch CUDA composition (bit-exact, NaN bytes included),
    both in the scale format `scale_fmt`.  An int8 y: int8_source_oracle.assert_exact."""
    if dst_dtype == torch.int8:
        int8_source_oracle.assert_exact(y, ys, x, g)
        return
    if scale_fmt is None:
        want_q, want_s = oracle_quantize(x.float().numpy(), g)
    else:
        want_q, want_s = ue8m0_oracle.quantize(x.float().numpy(), g, scale_fmt=scale_fmt)
    q, s = y.view(torch.uint8).cpu().numpy(), ys.cpu().numpy()
    if g == "block":
        assert_block_fp8_equal(q, s, want_q, want_s)
    else:
        assert_scaled_fp8_equal(q, s, want_q, np.asarray(want_s, np.float32), g)
    if scale_fmt is not None:
        want_q, want_s = ue8m0_oracle.torch_quantize(x.to(DEV), g, scale_fmt=scale_fmt)
        want_s = want_s.reshape(ys.shape)
        assert torch.equal(y.view(torch.uint8), want_q.view(torch.uint8))  # NaN bytes included
        nan = torch.isnan(want_s)
        assert torch.equal(torch.isnan(ys), nan) and torch.equal(ys.view(torch.int32)[~nan], want_s.view(torch.int32)[~nan])
        ue8m0_oracle.assert_pow2_over(ys, ue8m0_oracle.torch_quantize(x.to(DEV), g)[1])
    elif g == "block":
        bq_gpu.assert_torch_cuda(y, ys, x)
    else:
        sq_gpu.assert_torch_cuda(y, ys, x, g)


# ---- the regimes ------------------------------------------------------------------------------------
VARIANTS = ("finite", "special", "near_top", "update")


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("regime", sorted(REGIMES))
def test_regime_on_the_h100(regime, variant):
    run_regime(regime, variant)


def run_regime(regime, variant, scale_fmt=None, dst_dtype=E4M3):
    """Pull the regime's workload in `variant` with the scale format `scale_fmt` into `dst_dtype` destinations,
    and check it (module doc)."""
    r = REGIMES[regime]
    w = WORKLOADS[r.workload]
    xs = inputs(r.workload, variant)
    where = f"{regime} ({r.doc}), {variant}, scale_fmt={scale_fmt}, {dst_dtype}: {w.describe()}"
    pulled = Pulled(w.pulls, xs, scale_fmt=scale_fmt, dst_dtype=dst_dtype)
    try:
        pulled.pull()
        tables, geom = pulled.live_tables()
        assert r.holds(tables, geom), f"not reached: {where}"
        with named(where):
            pulled.check(xs)
            if variant == "update":
                xs = [(rand_full(p.shape, getattr(torch, p.dtype), w.seed + 50 + i) * -0.5) for i, p in enumerate(w.pulls)]
                pulled.update(xs)
                before = pulled.plans()
                pulled.pull()
                assert pulled.plans() == before  # replayed, not rebuilt
                pulled.check(xs)
    finally:
        pulled.close()


# ---- a mixed-dtype dict -----------------------------------------------------------------------------
def mixed_pulls():
    """bf16, f16 and f32 names at every granularity; the f16 shards start 2 bytes past a 16-byte boundary."""
    shapes = {"block": ((200, 260), 0), "channel": ((130, 200), 1), "tensor": ((2, 100, 136), 1)}
    out = []
    for d in ES:
        for g in GRANULARITIES:
            shape, dim = shapes[g]
            out.append(Pull(d, shape, split(shape, 2, dim), whole(shape), g, (1, 1) if d == "float16" else ()))
    return out


def test_mixed_dtype_dict_pulls_and_replays():
    pulls = mixed_pulls()
    xs = [rand_full(p.shape, getattr(torch, p.dtype), 70 + i) for i, p in enumerate(pulls)]
    plain = (torch.randn(96, 80, generator=torch.Generator().manual_seed(71)) * 0.1).to(torch.bfloat16)
    cast = torch.randn(64, 48, generator=torch.Generator().manual_seed(72))
    src = DirectWeightSyncSource()
    h = src.register({"plain": plain.to(DEV), "cast": cast.to(DEV)}, rank=0)
    extra = {"plain": torch.zeros(96, 80, dtype=torch.bfloat16, device=DEV), "cast": torch.zeros(64, 48, dtype=torch.bfloat16, device=DEV)}
    pulled = Pulled(pulls, xs, {"plain": [h["plain"]], "cast": [h["cast"]]}, extra)
    try:
        pulled.pull()
        tables, _ = pulled.live_tables()
        assert {int(b["src_dtype"]) for b in tables.block[0]} == {_native.TSB_BF16, _native.TSB_F16, _native.TSB_F32}
        assert len(tables.scaled[0]) and len(tables.scaled[2])
        pulled.check(xs)
        assert torch.equal(extra["plain"].cpu(), plain) and torch.equal(extra["cast"], cast.to(DEV).to(torch.bfloat16))
        before = pulled.plans()
        pulled.update(xs)
        extra["plain"].zero_()
        extra["cast"].zero_()
        pulled.pull()
        assert pulled.plans() == before
        pulled.check(xs)
        assert torch.equal(extra["plain"].cpu(), plain) and torch.equal(extra["cast"], cast.to(DEV).to(torch.bfloat16))
    finally:
        pulled.close()
        run(src.cleanup())


# ---- past byte 2^32 ---------------------------------------------------------------------------------
def test_quantise_pull_past_byte_2_32():
    """A bf16 stack of 129 experts [4096, 8192]: its source (8.7 GB) and each fp8 destination (4.3 GB) run past
    byte 2^32; block, channel and tensor scales in turn, experts 0, 127 and 128 against torch CUDA."""
    shape = (129, 4096, 8192)
    n = int(np.prod(shape))
    assert n > 2**32
    skip_unless_free(3 * n)  # the bf16 source and one fp8 destination
    gen = torch.Generator(DEV).manual_seed(6)
    x = torch.empty(shape, dtype=torch.bfloat16, device=DEV)
    for e in range(shape[0]):
        x[e] = torch.randn(shape[1:], device=DEV, generator=gen) * (0.01 * (1 + e % 5))
    src = DirectWeightSyncSource()
    try:
        h = src.register({"w": x}, rank=0)["w"]
        for g in GRANULARITIES:
            qb, q = guarded(shape, E4M3)
            sb, s = guarded(scale_shape(g, shape), torch.float32)
            sync = DirectWeightSyncDest()
            run(sync.pull({"w": [h]}, {"w": q}, **{KW[g]: {"w": s}}))
            for e in (0, 127, 128):
                want_q, want_s = block_fp8_oracle.torch_quantize(x[e]) if g == "block" else scaled_fp8_oracle.torch_quantize(x[e], g)
                assert torch.equal(q[e].view(torch.uint8), want_q.view(torch.uint8)), (g, e)
                assert torch.equal(s[e].reshape(-1).view(torch.int32), want_s.reshape(-1).view(torch.int32)), (g, e)
            assert guards_intact(qb) and guards_intact(sb), g
            sync.close()
            del q, s, qb, sb, sync
            torch.cuda.empty_cache()
    finally:
        run(src.cleanup())
        del x
        torch.cuda.empty_cache()


# ---- random layouts with special values -------------------------------------------------------------
def boundary_spots(p: Pull, rng: random.Random, k: int = 8):
    """`k` global coordinates of the window drawn from the corners of every shard inside it, the rows and
    columns around block edges, and the ends and starts of consecutive rows."""
    (doff, dloc) = p.dst
    cands = []
    for off, loc in p.src:
        lo = [max(a, b) for a, b in zip(off, doff)]
        hi = [min(a + m, b + n) for a, m, b, n in zip(off, loc, doff, dloc)]
        if any(a >= b for a, b in zip(lo, hi)):
            continue
        lead = tuple(lo[:-2])
        for r in (lo[-2], hi[-2] - 1):
            for c in (lo[-1], hi[-1] - 1):
                cands.append(lead + (r, c))
    *lo, r0, c0 = doff
    *ln, n, kk = dloc
    for rr in (BLOCK - 1, BLOCK, rng.randrange(n)):
        for cc in (BLOCK - 1, BLOCK, 15, 16, kk - 1, 0):
            if rr < n and cc < kk:
                cands.append(tuple(o + rng.randrange(m) for o, m in zip(lo, ln)) + (r0 + rr, c0 + cc))
    return rng.sample(cands, min(k, len(cands)))


def plant_random(x, p: Pull, rng: random.Random, seed: int):
    """NaN, +-Inf, -0, a subnormal and the dtype's top at boundary spots; one group all zero, one subnormal."""
    x = x.float().clone()
    tiny = torch.finfo(getattr(torch, p.dtype)).tiny
    values = (float("nan"), float("inf"), float("-inf"), -0.0, tiny * 0.25, TOP[p.dtype])
    for j, c in enumerate(boundary_spots(p, rng)):
        x[c] = values[(j + seed) % len(values)]
    for j, kind in enumerate(("zero", "subnormal")):
        c = tuple(o + rng.randrange(m) for o, m in zip(*p.dst))
        fill_group(x, p, group_of(p, c), kind, seed + j)
    return x.to(getattr(torch, p.dtype))


@pytest.mark.parametrize("seed", range(24))
def test_random_layouts_with_special_values(seed):
    run_random_layout(seed)


def run_random_layout(seed, dst_dtype=E4M3):
    """Pull the layout drawn from `seed`, with special values, into a `dst_dtype` destination and check it."""
    rng = random.Random(19000 + seed)
    w = draw(rng, "quant", seed)
    p = Pull(("bfloat16", "float16", "float32")[seed % 3], w.shape, w.src, w.dst, w.out)
    x = plant_random(torch.randn(w.shape, generator=torch.Generator().manual_seed(seed)) * 0.05, p, rng, seed)
    pulled = Pulled((p,), [x], dst_dtype=dst_dtype)
    try:
        with named(f"seed {seed}: {p.describe()}"):
            pulled.pull()
            pulled.live_tables()
            pulled.check([x])
    finally:
        pulled.close()

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

import random
from functools import partial

import numpy as np
import pytest
import torch

from oracle import block_fp8_oracle, scaled_fp8_oracle
from oracle.dequant_fp8_oracle import DST, torch_dequantize
from oracle.requant_fp8_oracle import torch_requantize
from tests.fp8_regimes import (REGIMES, VARIANTS, Workload, assert_dequant_oracle, assert_dequant_torch_cuda,
                               assert_requant_oracle, assert_requant_torch_cuda, draw, run_regime, want_bits, whole)
from tests.helpers import (DEV, E4M3, KW, cleanup, dest_scale_shape, guarded, guards_intact, named, native_session,
                           pull_box, region, register_boxes, run, skip_unless_free)
from tests.test_dequant_fp8_cpu import local_scale
from tests.test_requant_fp8_cpu import fp8_full, global_scale
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource
from torchstore_b200.transport.types import TensorSlice

pytestmark = pytest.mark.gpu
_init = pytest.fixture(scope="module", autouse=True)(native_session)


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("regime", sorted(REGIMES))
def test_regime_on_the_h100(regime, variant):
    run_regime(regime, variant)


# ---- past byte 2^32 ---------------------------------------------------------------------------------
def big_stack(experts, rows, cols, seed):
    """A finite fp8 MoE stack on the GPU, one expert at a time (no full-size temporary)."""
    gen = torch.Generator(DEV).manual_seed(seed)
    q = torch.empty(experts, rows, cols, dtype=torch.uint8, device=DEV)
    for e in range(experts):
        b = torch.randint(0, 0x7F, (rows, cols), dtype=torch.uint8, device=DEV, generator=gen)  # 0x00..0x7E: finite
        q[e] = b | (torch.randint(0, 2, (rows, cols), dtype=torch.uint8, device=DEV, generator=gen) << 7)
    return q.view(E4M3)


def test_requantise_past_byte_2_32():
    """A block-scaled fp8 stack of 129 experts [4096, 8192] (4.3 GB) into a per-channel destination: the source
    shard and the destination both run past byte 2^32; the last matrices against the torch CUDA composition."""
    shape = (129, 4096, 8192)
    n = int(np.prod(shape))
    assert n > 2**32
    skip_unless_free(2 * n)
    q = big_stack(*shape, seed=1)
    s = global_scale("block", shape, 1).to(DEV)
    sources, handles = register_boxes(q, [whole(shape)], granularity="block", scale_of=partial(local_scale, s, "block"))
    sync, y, ys, bases = pull_box(handles, shape, whole(shape), E4M3, granularity="channel", requantize=True)
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
    sources, handles = register_boxes(q, [whole(shape)], granularity="channel",
                                      scale_of=partial(local_scale, s, "channel"))
    sync, y, _, (base,) = pull_box(handles, shape, whole(shape), torch.bfloat16)
    for e in (0, shape[0] - 2, shape[0] - 1):
        assert torch.equal(y[e], torch_dequantize(q[e], s[e], "channel")), e
    assert guards_intact(base)
    sync.close()
    cleanup(sources)
    del q, y, base, sources, handles
    torch.cuda.empty_cache()


# ---- random layouts across the four scaled plan kinds ----------------------------------------------
class Case:
    """One name of a pull drawn by draw(): its sources, its destination and its check."""

    def __init__(self, name: str, w: Workload):
        self.name, self.w = name, w
        self.scale = self.y_scale = None
        if w.kind == "quant":
            self.x = (torch.randn(w.shape, generator=torch.Generator().manual_seed(w.seed)) * 0.05).to(getattr(torch, w.sg))
            self.sources, self.handles = register_boxes(self.x, list(w.src), name=name)
        else:
            self.q, self.scale = fp8_full(w.shape, w.seed), global_scale(w.sg, w.shape, w.seed)
            self.sources, self.handles = register_boxes(self.q, list(w.src), name=name, granularity=w.sg,
                                                        scale_of=partial(local_scale, self.scale, w.sg))
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
            assert_dequant_oracle(self.y, want_bits(self.q, self.scale, w.sg, w.dst, DST[w.out]))
            assert_dequant_torch_cuda(self.y, self.q, self.scale, w.sg, w.dst)
        else:
            assert_requant_oracle(self.y, self.y_scale, self.q, self.scale, w.sg, w.dst, w.out)
            assert_requant_torch_cuda(self.y, self.y_scale, self.q, self.scale, w.sg, w.dst, w.out)
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

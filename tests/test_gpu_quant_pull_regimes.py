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

import numpy as np
import pytest
import torch

from oracle import block_fp8_oracle, scaled_fp8_oracle
from tests.fp8_regimes import split, whole
from tests.helpers import (DEV, E4M3, KW, dest_scale_shape, guarded, guards_intact, native_session, rand_full, run,
                           skip_unless_free)
from tests.quant_pull_regimes import (ES, GRANULARITIES, REGIMES, VARIANTS, Pull, Pulled, run_random_layout,
                                      run_regime)
from torchstore_b200 import _native
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource

pytestmark = pytest.mark.gpu
_init = pytest.fixture(scope="module", autouse=True)(native_session)


# ---- the regimes ------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("regime", sorted(REGIMES))
def test_regime_on_the_h100(regime, variant):
    run_regime(regime, variant)


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
            sb, s = guarded(dest_scale_shape(g, shape), torch.float32)
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


@pytest.mark.parametrize("seed", range(24))
def test_random_layouts_with_special_values(seed):
    run_random_layout(seed)

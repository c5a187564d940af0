"""Source-side quantisation on the H100 in every regime of tests/source_quant_regimes.py, with special values,
past byte 2^32, behind work queued on the caller's stream, and through every consumer of handles whose shards
carry their own scales.

* Regimes: every catalogue workload registered through ``DirectWeightSyncSource.register(quantize=...)`` with
  finite data, with Inf / -Inf, NaN, all-zero or subnormal values in the first and last group of every
  target, and after an in-place update and ``refresh()``; the regime asserted again from the tables of the
  live addresses (and their size against plan_info); bit-exact against torch CUDA (NaN bytes included) and the
  numpy oracle on finite groups.  Each workload is also driven through Plans.build_source_quant on guarded
  buffers.  The regime runners take the staging dtype (``quant_dtype``, float8_e4m3fn by default; int8 staging is
  checked against oracle/int8_source_oracle.py and its torch rendering).
* The torch CPU fixture (tests/golden/source_quant_vectors.npz) on the device, at its recorded offsets.
* Consumers: dequantising, requantising and raw fp8 pulls of source-quantised shards that hold different scales
  for the groups they share (column shards, 2-D meshes, EP x FSDP x TP, replicas), against per-shard references.
* Seeded random round trips (a layout, a dtype, a granularity and a consumer with its window), and mixed
  registers of several quantised names and a transfer_dtype name refreshed with changed weights."""

import random

import numpy as np
import pytest
import torch

from oracle.source_quant_oracle import GRANULARITIES, fixture_inputs, synth_f32, torch_quantize
from tests.fp8_regimes import split, whole
from tests.helpers import (DEV, E4M3, cleanup, guarded, guards_intact, named, native_session, pull_box, region, register_boxes, run,
                           shard_box, skip_unless_free)
from tests.source_quant_regimes import (REGIMES, VARIANTS, WORKLOADS, assert_exact, local_slice, run_guarded,
                                        run_regime)
from tests.test_source_quant_cpu import assert_source_quant_equal, fixture_cases
from tests.test_source_quant_regimes_cpu import (CONSUMERS, SHARD_LAYOUTS, assert_shared_groups_differ, layout_shards,
                                                 oracle_shards, want_consumer, windows)
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource
from torchstore_b200.transport.types import TensorSlice

pytestmark = pytest.mark.gpu
_init = pytest.fixture(scope="module", autouse=True)(native_session)


# ---- the regimes ------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("regime", sorted(REGIMES))
def test_regime_on_the_h100(regime, variant):
    run_regime(regime, variant)


@pytest.mark.parametrize("name", sorted(WORKLOADS))
def test_workload_writes_nothing_outside_its_outputs(name):
    """The workload's plan driven directly on guarded fp8 and scale buffers, launched twice."""
    run_guarded(name)


# ---- the torch CPU fixture on the device ------------------------------------------------------------
INPUTS = {name: x for name, x, *_ in fixture_inputs()}


@pytest.mark.parametrize("case", fixture_cases(), ids=lambda c: c[0])
def test_fixture_on_the_h100(case):
    name, _, g, r0, c0, want_q, want_s = case
    x = INPUTS[name]
    src = DirectWeightSyncSource()
    src.register({"w": x.to(DEV)}, rank=0, tensor_slices={"w": local_slice(x.shape, r0, c0)}, quantize={"w": g})
    q, s, _ = src._quantized["w"]
    assert_source_quant_equal(q.view(torch.uint8).cpu().numpy(), s.cpu().numpy(), want_q, want_s, g, r0, c0)
    run(src.cleanup())


# ---- consumers of shard-local scales ----------------------------------------------------------------
def assert_staging_is_the_oracle(sources, shards, name="w"):
    for (src, *_), (off, loc, want_q, want_s) in zip(sources, shards):
        q, s, _ = src._quantized[name]
        assert np.array_equal(q.view(torch.uint8).cpu().numpy(), want_q), off
        assert np.array_equal(s.cpu().numpy().view(np.uint32), want_s.view(np.uint32)), off


def pull_consumer(handles, shape, g, consumer, window):
    """One pull of `handles` into a guarded window -> (result, want) as comparable numpy arrays, guards intact."""
    if consumer in GRANULARITIES:
        sync, y, ys, bases = pull_box(handles, shape, window, E4M3, granularity=consumer, requantize=True)
        got = (y.view(torch.uint8).cpu().numpy(), ys.cpu().numpy().reshape(-1).view(np.uint32))
    elif consumer == "raw":
        base, y = guarded(window[1], E4M3)
        sync, bases = DirectWeightSyncDest(), (base,)
        run(sync.pull({"w": handles}, {"w": y}, {"w": TensorSlice(window[0], (0,), shape, window[1], (1,))}))
        got = y.view(torch.uint8).cpu().numpy()
    else:
        sync, y, _, bases = pull_box(handles, shape, window, getattr(torch, consumer))
        got = y.view(torch.int16 if y.element_size() == 2 else torch.int32).cpu().numpy()
    assert all(guards_intact(b) for b in bases)
    sync.close()
    return got


def assert_consumer(got, want, consumer):
    if consumer in GRANULARITIES:
        assert np.array_equal(got[0], want[0])
        assert np.array_equal(got[1], np.asarray(want[1], np.float32).reshape(-1).view(np.uint32))
    else:
        assert np.array_equal(got.view(want.dtype), want)


@pytest.mark.parametrize("g", GRANULARITIES)
@pytest.mark.parametrize("layout", sorted(SHARD_LAYOUTS))
def test_consumers_of_shard_local_scales(layout, g):
    shape, boxes, x, shards = layout_shards(layout, g, 300 + len(layout))
    assert_shared_groups_differ(shards, g)
    sources, handles = register_boxes(x, boxes, quantize={"w": g})
    try:
        assert_staging_is_the_oracle(sources, shards)
        for consumer, win in CONSUMERS:
            window = windows(shape)[win]
            with named(f"{layout} {g} -> {consumer} over the {win} window"):
                assert_consumer(pull_consumer(handles, shape, g, consumer, window),
                                want_consumer(shape, shards, g, consumer, window), consumer)
    finally:
        cleanup(sources)


# ---- seeded random round trips ----------------------------------------------------------------------
WIDTHS = (16, 24, 64, 130, 260, 520, 16384, 16385, 32784)
DTYPES = (torch.bfloat16, torch.float16, torch.float32)
CONSUMER_KINDS = ("bfloat16", "float16", "float32", "block", "channel", "tensor", "raw")


def draw(rng: random.Random):
    """A global shape, a source dtype, a granularity, source boxes and a consumer with its window."""
    k = rng.choice(WIDTHS)
    n = rng.randint(1, max(1, min(300, 400_000 // k)))
    shape = (rng.randint(2, 4), n, k) if rng.random() < 0.3 else (n, k)
    layout = rng.choice(["rows", "cols", "2d", "replica"] + ["ep"] * (len(shape) == 3))
    if layout == "rows":
        boxes = split(shape, rng.randint(2, 5), -2)
    elif layout == "cols":
        boxes = split(shape, rng.randint(2, 4), -1)
    elif layout == "2d":
        rows, cols = split(shape, rng.randint(2, 3), -2), split(shape, 2, -1)
        boxes = tuple((ro[:-1] + (co[-1],), rl[:-1] + (cl[-1],)) for ro, rl in rows for co, cl in cols)
    elif layout == "replica":
        boxes = split(shape, 2, -2) * 2
    else:
        boxes = split(shape, shape[0], 0)
    boxes = tuple(b for b in boxes if 0 not in b[1])
    tp = rng.choice(["whole", "rows", "cols"])
    window = whole(shape) if tp == "whole" else shard_box(shape, 2, rng.randint(0, 1), len(shape) - (2 if tp == "rows" else 1))
    if 0 in window[1]:
        window = whole(shape)
    return shape, rng.choice(DTYPES), rng.choice(GRANULARITIES), layout, boxes, rng.choice(CONSUMER_KINDS), window


@pytest.mark.parametrize("seed", range(36))
def test_random_round_trips(seed):
    rng = random.Random(11000 + seed)
    shape, dtype, g, layout, boxes, consumer, window = draw(rng)
    x = (torch.randn(shape, generator=torch.Generator().manual_seed(seed)) * 0.05).to(dtype)
    shards = oracle_shards(x, g, boxes)
    sources, handles = register_boxes(x, boxes, quantize={"w": g})
    try:
        with named(f"seed {seed}: {str(dtype)[6:]}{list(shape)} {g} {layout} {[b for b in boxes]} -> {consumer} {window}"):
            for (src, *_), (off, loc) in zip(sources, boxes):
                q, s, _ = src._quantized["w"]
                assert_exact(q, s, region(x, off, loc).contiguous(), g, off[-2], off[-1])
            assert_consumer(pull_consumer(handles, shape, g, consumer, window), want_consumer(shape, shards, g, consumer, window),
                            consumer)
    finally:
        cleanup(sources)


@pytest.mark.parametrize("seed", range(6))
def test_random_mixed_registers_refresh_twice(seed):
    """Two ranks, each registering three quantised names of different dtypes and granularities and one
    transfer_dtype name in one register(); the weights change in place and refresh() runs twice; then every
    quantised name is dequantised into f32 by one pull."""
    rng = random.Random(12000 + seed)
    names = {}
    for name, dtype in zip("abc", rng.sample(DTYPES, 3)):
        k = rng.choice(WIDTHS[:6] + (16385,))
        names[name] = ((rng.randint(2, 3), rng.randint(2, 140), k) if rng.random() < 0.3 else (rng.randint(2, 300), k), dtype,
                       rng.choice(GRANULARITIES))
    plain = (64, rng.choice((48, 130)))
    boxes = {n: split(shape, 2, -2) for n, (shape, _, _) in names.items()}
    full = {n: (torch.randn(shape, generator=torch.Generator().manual_seed(100 * seed + i)) * 0.05).to(dtype)
            for i, (n, (shape, dtype, _)) in enumerate(names.items())}
    sources, locals_, handles = [], [], {n: [] for n in names}
    for r in range(2):
        sd = {n: region(full[n], *boxes[n][r]).contiguous().to(DEV) for n in names}
        sd["p"] = torch.randn(plain, device=DEV)
        slices = {n: TensorSlice(boxes[n][r][0], (r,), tuple(names[n][0]), boxes[n][r][1], (2,)) for n in names}
        src = DirectWeightSyncSource()
        h = src.register(sd, rank=r, transfer_dtype=torch.bfloat16, tensor_slices=slices,
                         quantize={n: names[n][2] for n in names})
        for n in names:
            handles[n].append(h[n])
        sources.append(src)
        locals_.append(sd)
    try:
        for step in range(2):
            for r, sd in enumerate(locals_):
                for n, t in sd.items():
                    t.mul_(-0.5 if step else 3.0).add_(0.001 * (r + 1))
                assert sources[r].refresh() == 4
                for n in names:
                    q, s, _ = sources[r]._quantized[n]
                    off = boxes[n][r][0]
                    with named(f"seed {seed} step {step} rank {r} {n}: {names[n]}"):
                        assert_exact(q, s, sd[n], names[n][2], off[-2], off[-1])
                staging, local = sources[r]._staging["p"]
                assert torch.equal(staging, local.to(torch.bfloat16))
        for n, (shape, _, g) in names.items():
            shards = oracle_shards(torch.cat([sd[n].cpu() for sd in locals_], dim=-2), g, boxes[n])
            with named(f"seed {seed} pull {n}: {names[n]}"):
                assert_consumer(pull_consumer(handles[n], shape, g, "float32", whole(shape)),
                                want_consumer(shape, shards, g, "float32", whole(shape)), "float32")
    finally:
        for src in sources:
            run(src.cleanup())


# ---- past byte 2^32 ---------------------------------------------------------------------------------
def test_quantise_past_byte_2_32():
    """A bf16 stack of 129 experts [4096, 8192]: its source (8.7 GB) and fp8 staging (4.3 GB) both run past byte
    2^32; each granularity in turn, experts 0, 127 and 128 against torch CUDA."""
    shape = (129, 4096, 8192)
    n = int(np.prod(shape))
    assert n > 2**32
    skip_unless_free(3 * n + 2**30)
    gen = torch.Generator(DEV).manual_seed(5)
    x = torch.empty(shape, dtype=torch.bfloat16, device=DEV)
    for e in range(shape[0]):
        x[e] = torch.randn(shape[1:], device=DEV, generator=gen) * (0.01 * (1 + e % 5))
    try:
        for g in GRANULARITIES:
            src = DirectWeightSyncSource()
            src.register({"w": x}, rank=0, quantize={"w": g})
            q, s, _ = src._quantized["w"]
            for e in (0, 127, 128):
                want_q, want_s = torch_quantize(x[e], g)
                assert torch.equal(q[e].view(torch.uint8), want_q.view(torch.uint8)), (g, e)
                assert torch.equal(s[e].reshape(-1).view(torch.int32), want_s.reshape(-1).view(torch.int32)), (g, e)
            run(src.cleanup())
            del q, s, src
            torch.cuda.empty_cache()
    finally:
        del x
        torch.cuda.empty_cache()


# ---- ordering against the caller's stream -----------------------------------------------------------
@pytest.mark.parametrize("stream", ("current", "side"))
def test_refresh_quantises_what_the_callers_stream_just_wrote(stream):
    """The weight update is queued behind a ~50 ms spin on the caller's current stream (the default one, or a
    side stream made current); refresh() must wait for it and quantise the updated weights."""
    old = synth_f32((512, 640), 61).to(torch.bfloat16).to(DEV)
    new = (synth_f32((512, 640), 62) * 3).to(torch.bfloat16).to(DEV)
    sources = []
    for g in GRANULARITIES:
        src = DirectWeightSyncSource()
        w = old.clone()
        src.register({"w": w}, rank=0, quantize={"w": g})
        sources.append((src, w, g))
    torch.cuda.synchronize()
    s = torch.cuda.current_stream() if stream == "current" else torch.cuda.Stream()
    try:
        with torch.cuda.stream(s):
            for src, w, g in sources:
                torch.cuda._sleep(100_000_000)
                w.copy_(new)
                assert src.refresh() == 1
                q, sc, _ = src._quantized["w"]
                assert_exact(q, sc, new, g, 0, 0)
    finally:
        torch.cuda.synchronize()
        for src, _, _ in sources:
            run(src.cleanup())

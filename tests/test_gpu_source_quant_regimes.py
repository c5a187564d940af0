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

import asyncio
import random

import numpy as np
import pytest
import torch

from oracle import int8_source_oracle
from oracle.source_quant_oracle import GRANULARITIES, fixture_inputs, synth_f32, torch_quantize
from tests import test_gpu_dequant_fp8 as dq_gpu
from tests import test_gpu_requant_fp8 as rq_gpu
from tests.fp8_regimes import split, whole
from tests.helpers import region, shard_box
from tests.source_quant_regimes import CODE, REGIMES, WORKLOADS, Target, plan_bytes
from tests.test_gpu_dequant_fp8 import guarded, guards_intact
from tests.test_gpu_fp8_regimes import named, skip_unless_free
from tests.test_gpu_source_quant import assert_exact
from tests.test_source_quant_cpu import CODE as GCODE
from tests.test_source_quant_cpu import assert_source_quant_equal, compile_host, fixture_cases
from tests.test_source_quant_regimes_cpu import (CONSUMERS, SHARD_LAYOUTS, assert_shared_groups_differ, layout_shards,
                                                 oracle_shards, want_consumer, windows, workload_inputs)
from torchstore_b200 import _native
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource, source_scale_shapes
from torchstore_b200.launch import Plans
from torchstore_b200.transport.types import TensorSlice

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
E4M3 = torch.float8_e4m3fn


@pytest.fixture(scope="module", autouse=True)
def _init():
    _native.init()
    yield


def run(coro):
    return asyncio.run(coro)


def on_device(x: torch.Tensor, misalign: int = 0) -> torch.Tensor:
    """`x` on the GPU, starting `misalign` elements into a fresh allocation (not 16-byte aligned if > 0) with
    4096 elements of slack after it, so that reads past a shard's end stay inside the allocation."""
    flat = torch.zeros(x.numel() + 4096, dtype=x.dtype, device=DEV)
    out = flat[misalign: misalign + x.numel()].view(x.shape)
    out.copy_(x.to(DEV))
    return out


def local_slice(shape, row0, col0, global_shape=None, rank=0, ranks=1):
    lead = tuple(shape[:-2])
    gshape = global_shape or lead + (row0 + shape[-2], col0 + shape[-1])
    offsets = (0,) * len(lead) + (row0, col0)
    return TensorSlice(offsets, (rank,), tuple(gshape), tuple(shape), (ranks,))


# ---- the regimes ------------------------------------------------------------------------------------
def group_boxes(t: Target):
    """Index tuples of the first and the last group of a target's shard."""
    *lead, n, k = t.shape
    first_m, last_m = (0,) * len(lead), tuple(e - 1 for e in lead)
    if t.granularity == "block":
        r1, c1 = min(n, 128 - t.row0 % 128), min(k, 128 - t.col0 % 128)
        lr, lc = max(0, (t.row0 + n - 1) // 128 * 128 - t.row0), max(0, (t.col0 + k - 1) // 128 * 128 - t.col0)
        return first_m + (slice(0, r1), slice(0, c1)), last_m + (slice(lr, n), slice(lc, k))
    if t.granularity == "channel":
        return first_m + (slice(0, 1), slice(None)), last_m + (slice(n - 1, n), slice(None))
    return first_m + (slice(None), slice(None)), last_m + (slice(None), slice(None))


def plant(x: torch.Tensor, t: Target, kind: str, seed: int) -> torch.Tensor:
    """Special values in the first and the last group of `x` (in its dtype): +Inf and -Inf, or NaN, at the
    first element of the first group and the last element of the last; or both groups all zero or subnormal."""
    x = x.float().clone()
    first, last = group_boxes(t)
    first_elem, last_elem = (0,) * len(t.shape), tuple(e - 1 for e in t.shape)
    if kind in ("inf", "nan"):
        x[first_elem] = float("inf") if kind == "inf" else float("nan")
        x[last_elem] = float("-inf") if kind == "inf" else float("nan")
    elif kind == "zero":
        x[first] = 0
        x[last] = 0
    elif kind == "subnormal":
        tiny = torch.finfo(getattr(torch, t.dtype)).tiny
        for box in (first, last):
            x[box] = synth_f32(tuple(x[box].shape), seed, spread=0) * tiny * 0.5
    return x.to(getattr(torch, t.dtype))


def register_workload(name, xs, scale_fmt=None, quant_dtype=None):
    """One register() of every target of workload `name` (values `xs`), in the scale format `scale_fmt` and the
    staging dtype `quant_dtype` -> (source, handles, device shards)."""
    w = WORKLOADS[name]
    src = DirectWeightSyncSource()
    sd, slices, quant = {}, {}, {}
    for i, (t, x) in enumerate(zip(w.targets, xs)):
        sd[f"t{i}"] = on_device(x, t.misalign)
        slices[f"t{i}"] = local_slice(t.shape, t.row0, t.col0)
        quant[f"t{i}"] = t.granularity
    handles = src.register(sd, rank=0, tensor_slices=slices, quantize=quant, scale_fmt=scale_fmt, quant_dtype=quant_dtype)
    return src, handles, sd


def live_tables(src, handles, w, quant_dtype=None):
    """Compile on the host the targets register() built, from the staging it allocated and the handles'
    offsets (for int8 staging with TSB_I8); check their size against plan_info -> (tables, targets)."""
    targets = []
    for i, t in enumerate(w.targets):
        fp8, scale, local = src._quantized[f"t{i}"]
        buf = handles[f"t{i}"].rdma_buffer
        rows, cols = local.shape[-2:]
        targets.append(_native.SourceQuantTarget(local.data_ptr(), fp8.data_ptr(), scale.data_ptr(), local.numel() // (rows * cols),
                                                 rows, cols, buf.row0, buf.col0, CODE[t.dtype], GCODE[t.granularity]))
    if quant_dtype == torch.int8:
        arr = _native.make_source_quant_target_array(len(targets))
        for i, t in enumerate(targets):
            arr[i] = t
        tables = _native.source_quant_compile_host(0, arr, len(targets), dst_dtype=_native.TSB_I8)
    else:
        tables = compile_host(targets)
    info = _native.plan_info(src._quant_plans[0])
    assert (info.num_tiles, info.src_bytes) == plan_bytes(tables)
    return tables, targets


def check_staging(src, w, xs, scale_fmt=None, quant_dtype=None):
    for i, (t, x) in enumerate(zip(w.targets, xs)):
        q, s, _ = src._quantized[f"t{i}"]
        with named(t.describe()):
            if quant_dtype == torch.int8:
                int8_source_oracle.assert_exact(q, s, x, t.granularity, t.row0, t.col0)
            else:
                assert_exact(q, s, x, t.granularity, t.row0, t.col0, scale_fmt)


VARIANTS = ("finite", "inf", "nan", "zero", "subnormal", "refresh")


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("regime", sorted(REGIMES))
def test_regime_on_the_h100(regime, variant):
    run_regime(regime, variant)


def run_regime(regime, variant, scale_fmt=None, quant_dtype=None):
    """Register the regime's workload in `variant` with the scale format `scale_fmt` and the staging dtype
    `quant_dtype`, and check it (module doc)."""
    r = REGIMES[regime]
    w = WORKLOADS[r.workload]
    xs = workload_inputs(r.workload)
    if variant not in ("finite", "refresh"):
        xs = [plant(x, t, variant, w.seed + i) for i, (t, x) in enumerate(zip(w.targets, xs))]
    src, handles, sd = register_workload(r.workload, xs, scale_fmt, quant_dtype)
    where = f"{regime} ({r.doc}), {variant}, scale_fmt={scale_fmt}, quant_dtype={quant_dtype}: {w.describe()}"
    try:
        tables, targets = live_tables(src, handles, w, quant_dtype)
        assert r.holds(tables, targets), f"not reached: {where}"
        with named(where):
            check_staging(src, w, xs, scale_fmt, quant_dtype)
            if variant == "refresh":
                xs = [synth_f32(t.shape, w.seed + 50 + i).to(x.dtype) * 0.25 for i, (t, x) in enumerate(zip(w.targets, xs))]
                for i, x in enumerate(xs):
                    sd[f"t{i}"].copy_(x.to(DEV))
                assert src.refresh() == len(w.targets)
                check_staging(src, w, xs, scale_fmt, quant_dtype)
    finally:
        run(src.cleanup())


@pytest.mark.parametrize("name", sorted(WORKLOADS))
def test_workload_writes_nothing_outside_its_outputs(name):
    """The workload's plan driven directly on guarded fp8 and scale buffers, launched twice."""
    run_guarded(name)


def run_guarded(name, scale_fmt=None, quant_dtype=None):
    w = WORKLOADS[name]
    xs = workload_inputs(name)
    targets, outs = [], []
    for t, x in zip(w.targets, xs):
        sv = on_device(x, t.misalign)
        sshape = source_scale_shapes(t.granularity, t.shape, t.row0, t.col0)[0]
        qbase, q = guarded(t.shape, quant_dtype or E4M3)
        sbase, s = guarded(sshape, torch.float32)
        rows, cols = t.shape[-2:]
        targets.append(_native.SourceQuantTarget(sv.data_ptr(), q.data_ptr(), s.data_ptr(), x.numel() // (rows * cols), rows, cols,
                                                 t.row0, t.col0, CODE[t.dtype], GCODE[t.granularity]))
        outs.append((sv, q, s, qbase, sbase))
    plans = Plans.build_source_quant({0: targets}, _native.TSB_QUANT_UE8M0 if scale_fmt else 0,
                                     _native.TSB_I8 if quant_dtype == torch.int8 else _native.TSB_F8E4M3)
    try:
        for _ in range(2):
            plans.launch()
            plans.synchronize()
    finally:
        plans.close()
    for t, x, (_, q, s, qbase, sbase) in zip(w.targets, xs, outs):
        with named(f"{name}: {t.describe()}"):
            if quant_dtype == torch.int8:
                int8_source_oracle.assert_exact(q, s, x, t.granularity, t.row0, t.col0)
            else:
                assert_exact(q, s, x, t.granularity, t.row0, t.col0, scale_fmt)
            assert guards_intact(qbase) and guards_intact(sbase)


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
def register_boxes(x_full, g, boxes, name="w"):
    """One source per box of `x_full`, quantised on registration -> (sources, handles)."""
    sources, handles = [], []
    for r, (off, loc) in enumerate(boxes):
        src = DirectWeightSyncSource()
        sl = TensorSlice(off, (r,), tuple(x_full.shape), loc, (len(boxes),))
        handles.append(src.register({name: region(x_full, off, loc).contiguous().to(DEV)}, rank=r, tensor_slices={name: sl},
                                    quantize={name: g})[name])
        sources.append(src)
    return sources, handles


def assert_staging_is_the_oracle(sources, shards, name="w"):
    for src, (off, loc, want_q, want_s) in zip(sources, shards):
        q, s, _ = src._quantized[name]
        assert np.array_equal(q.view(torch.uint8).cpu().numpy(), want_q), off
        assert np.array_equal(s.cpu().numpy().view(np.uint32), want_s.view(np.uint32)), off


def pull_consumer(handles, shape, g, consumer, window):
    """One pull of `handles` into a guarded window -> (result, want) as comparable numpy arrays, guards intact."""
    if consumer in GRANULARITIES:
        sync, y, ys, bases = rq_gpu.pull_into(handles, shape, window, consumer)
        got = (y.view(torch.uint8).cpu().numpy(), ys.cpu().numpy().reshape(-1).view(np.uint32))
    elif consumer == "raw":
        base, y = guarded(window[1], E4M3)
        sync, bases = DirectWeightSyncDest(), (base,)
        run(sync.pull({"w": handles}, {"w": y}, {"w": TensorSlice(window[0], (0,), shape, window[1], (1,))}))
        got = y.view(torch.uint8).cpu().numpy()
    else:
        sync, y, base = dq_gpu.pull_into(handles, shape, window, getattr(torch, consumer))
        bases = (base,)
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
    sources, handles = register_boxes(x, g, boxes)
    try:
        assert_staging_is_the_oracle(sources, shards)
        for consumer, win in CONSUMERS:
            window = windows(shape)[win]
            with named(f"{layout} {g} -> {consumer} over the {win} window"):
                assert_consumer(pull_consumer(handles, shape, g, consumer, window),
                                want_consumer(shape, shards, g, consumer, window), consumer)
    finally:
        for src in sources:
            run(src.cleanup())


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
    sources, handles = register_boxes(x, g, boxes)
    try:
        with named(f"seed {seed}: {str(dtype)[6:]}{list(shape)} {g} {layout} {[b for b in boxes]} -> {consumer} {window}"):
            for src, (off, loc) in zip(sources, boxes):
                q, s, _ = src._quantized["w"]
                assert_exact(q, s, region(x, off, loc).contiguous(), g, off[-2], off[-1])
            assert_consumer(pull_consumer(handles, shape, g, consumer, window), want_consumer(shape, shards, g, consumer, window),
                            consumer)
    finally:
        for src in sources:
            run(src.cleanup())


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

"""The INT8 kernels on the H100 in the regimes the fp8 suites reach, at the int8 rounding edges in every route, over
the INT8 golden fixtures, past byte 2^32 and across random layouts.

* Regimes: every regime of tests/quant_pull_regimes.py and tests/source_quant_regimes.py and the ``dq_*`` regimes of
  tests/fp8_regimes.py, in each catalogue's own variants, with int8 destinations, int8 staging or int8 handles; every
  source workload's plan also driven on guarded int8 buffers.  Each run re-asserts the regime from the live plan's
  tables (and their size against plan_info), is bit for bit the numpy oracle and the torch CUDA rendering (int8
  bytes everywhere, scale_inv NaN-agnostic only where it is NaN), and leaves the guard bytes intact.  The quantisers
  also hold the formula's invariants in every group: no -128, a non-finite group all zeros, and +-127 at the amax
  element of every finite group with amax >= 1e-4.
* Rounding edges, route by route: groups whose values are searched so that the formula ``rint(rn(x * rn(127 /
  amax_c)))`` and a named wrong rendering (``x / scale_inv``, ``x * rn(1 / scale_inv)``, the unrounded product,
  rounding half away from zero, truncation) give different bytes; ties k + 1/2 of both parities and signs; amaxes
  at the 1e-4 floor and 127 (scale exactly 1).  Each route asserts from its inputs that every rendering is told
  apart at least once.
* The fixtures tests/golden/int8_vectors.npz and tests/golden/int8_source_vectors.npz on the device, and every
  int8 value against int8_source_oracle.SCALE_SET.
* Past byte 2^32: an int8 quantising pull, int8 staging and an int8 dequantising pull of 129 x [4096, 8192] stacks.
* Random layouts: the quantising pull's random layouts with special values into int8 destinations, and the
  dequantising draws from int8 handles."""

import os
import random
from functools import partial

import numpy as np
import pytest
import torch

from oracle import int8_oracle as i8
from oracle import int8_source_oracle as i8s
from tests import fp8_regimes, quant_pull_regimes, source_quant_regimes
from tests.helpers import (DEV, I8, KW, cleanup, dest_scale_shape, guarded, guards_intact, named, native_session, pull_box,
                           register_boxes, run, skip_unless_free)
from tests.quant_pull_regimes import Pull, split, whole
from tests.test_dequant_fp8_cpu import local_scale as dq_local_scale
from tests.test_requant_fp8_cpu import global_scale
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource

pytestmark = pytest.mark.gpu
DTYPES = (torch.bfloat16, torch.float16, torch.float32)
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
DQ_REGIMES = sorted(n for n, r in fp8_regimes.REGIMES.items() if fp8_regimes.WORKLOADS[r.workload].kind == "dequant")
_init = pytest.fixture(scope="module", autouse=True)(native_session)


# ---- every regime in int8 ----------------------------------------------------------------------------
@pytest.mark.parametrize("variant", quant_pull_regimes.VARIANTS)
@pytest.mark.parametrize("regime", sorted(quant_pull_regimes.REGIMES))
def test_quant_pull_regime(regime, variant):
    quant_pull_regimes.run_regime(regime, variant, dst_dtype=I8)


@pytest.mark.parametrize("variant", source_quant_regimes.VARIANTS)
@pytest.mark.parametrize("regime", sorted(source_quant_regimes.REGIMES))
def test_source_regime(regime, variant):
    source_quant_regimes.run_regime(regime, variant, quant_dtype=I8)


@pytest.mark.parametrize("name", sorted(source_quant_regimes.WORKLOADS))
def test_source_workload_writes_nothing_outside_its_outputs(name):
    source_quant_regimes.run_guarded(name, quant_dtype=I8)


@pytest.mark.parametrize("variant", fp8_regimes.VARIANTS)
@pytest.mark.parametrize("regime", DQ_REGIMES)
def test_dequant_regime(regime, variant):
    fp8_regimes.run_regime(regime, variant, src_dtype=I8)


# ---- the rounding edges, route by route ----------------------------------------------------------------
N_GROUPS = 16  # the groups of i8.edge_groups: three at the 1e-4 floor, 127 and twelve searched amaxes


def assert_told_apart(x, g, r0=0, c0=0):
    """Every wrong rendering differs from the formula somewhere in x, and ties of both parities and signs occur."""
    told, ties = i8.told_apart(x, g, r0, c0)
    assert told == set(i8.WRONG), sorted(told)
    assert ties == {(k, s) for k in ("even", "odd") for s in (1, -1)}, sorted(ties)


QUANT_ROUTES = {  # route -> (granularity, shape of G groups, kind of the pass the plan must hold)
    "block_kernel": ("block", lambda G: (128, 128 * G), "block"),
    "rows_kernel": ("channel", lambda G: (G, 160), "bands"),
    "tensor_two_pass": ("tensor", lambda G: (G, 16, 64), "tiles"),
    "long_row_channel_two_pass": ("channel", lambda G: (G, 16400), "tiles"),
}


def long_rows(shape, dtype):
    return (shape[0], 8200) if dtype == torch.float32 else shape  # over the 32 KiB row stage


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("route", sorted(QUANT_ROUTES))
def test_rounding_edges_of_a_quantising_pull(route, dtype):
    g, shape_of, kind = QUANT_ROUTES[route]
    shape = shape_of(N_GROUPS)
    if route.startswith("long_row"):
        shape = long_rows(shape, dtype)
    x, n = i8.plant_rounding_edges(shape, dtype, g)
    assert n >= N_GROUPS == len(i8.edge_groups(str(dtype)[6:]))
    assert_told_apart(x, g)
    name = str(dtype)[6:]
    p = Pull(name, shape, split(shape, 2, -1), whole(shape), g)
    pulled = quant_pull_regimes.Pulled((p,), [x], dst_dtype=I8)
    try:
        pulled.pull()
        tables, _ = pulled.live_tables()
        if kind == "block":
            assert tables.block is not None and len(tables.block[0])
        else:
            bands, _, tiles, _ = tables.scaled
            assert (len(bands) > 0 and len(tiles) == 0) if kind == "bands" else (len(tiles) > 0 and len(bands) == 0)
        with named(f"{route} {name}"):
            pulled.check([x])
    finally:
        pulled.close()


SOURCE_ROUTES = {  # route -> (granularity, shard shape of at least G groups at (37, 70), kind of pass)
    "block_units": ("block", lambda G: (300, 128 * (G // 3 + 1)), "units"),
    "channel_units": ("channel", lambda G: (G, 200), "units"),
    "tensor_tiles": ("tensor", lambda G: (G, 16, 64), "tiles"),
    "long_row_channel": ("channel", lambda G: (G, 16400), "tiles"),
}


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("route", sorted(SOURCE_ROUTES))
def test_rounding_edges_of_source_side_quantisation(route, dtype):
    g, shape_of, kind = SOURCE_ROUTES[route]
    shape = shape_of(N_GROUPS)
    if route.startswith("long_row"):
        shape = long_rows(shape, dtype)
    x, n = i8.plant_rounding_edges(shape, dtype, g, 37, 70)
    assert n >= N_GROUPS
    assert_told_apart(x, g, 37, 70)
    name = str(dtype)[6:]
    w = source_quant_regimes.Workload((source_quant_regimes.Target(name, shape, g, 37, 70),), 0)
    src, handles, _ = register_one(w, x)
    try:
        (units, tiles, _), _ = source_quant_regimes.live_tables(src, handles, w, I8)
        assert (len(units) > 0 and len(tiles) == 0) if kind == "units" else (len(tiles) > 0 and len(units) == 0)
        q, s, _ = src._quantized["t0"]
        with named(f"{route} {name}"):
            i8s.assert_exact(q, s, x, g, 37, 70)
    finally:
        run(src.cleanup())


def register_one(w, x):
    """register() of the one target of `w` (values x) with int8 staging -> (source, handles, device shards)."""
    t = w.targets[0]
    src = DirectWeightSyncSource()
    sd = {"t0": x.to(DEV)}
    handles = src.register(sd, rank=0, tensor_slices={"t0": source_quant_regimes.local_slice(t.shape, t.row0, t.col0)},
                           quantize={"t0": t.granularity}, quant_dtype=I8)
    return src, handles, sd


# ---- the fixtures on the device ----------------------------------------------------------------------
def int8_pull(x, g):
    """A quantising pull of the whole of x into guarded int8 and scale buffers -> (q, s)."""
    src = DirectWeightSyncSource()
    try:
        h = src.register({"w": x.to(DEV)}, rank=0)["w"]
        qb, q = guarded(tuple(x.shape), I8)
        sb, s = guarded(dest_scale_shape(g, tuple(x.shape)), torch.float32)
        sync = DirectWeightSyncDest()
        run(sync.pull({"w": [h]}, {"w": q}, **{KW[g]: {"w": s}}))
        assert sync._int8_block_plans or sync._int8_scaled_plans
        sync.close()
        assert guards_intact(qb) and guards_intact(sb)
    finally:
        run(src.cleanup())
    return q, s


PULL_CASES = i8.fixture_inputs()


@pytest.mark.parametrize("i", range(len(PULL_CASES)), ids=lambda i: PULL_CASES[i][0])
def test_int8_fixture_as_quantising_pulls(i):
    d = np.load(os.path.join(GOLDEN, "int8_vectors.npz"))
    name, x, g = PULL_CASES[i]
    q, s = int8_pull(x, g)
    assert i8.digest(q.view(torch.uint8).cpu().numpy()) == str(d[f"q_sha{i}"]), name
    assert i8.same_scales(s.cpu().numpy().reshape(d[f"s{i}"].shape), d[f"s{i}"]), name
    i8s.assert_exact(q, s, x, g)


SOURCE_CASES = i8s.quant_inputs()


@pytest.mark.parametrize("i", range(len(SOURCE_CASES)), ids=lambda i: SOURCE_CASES[i][0])
def test_int8_source_fixture_as_staging(i):
    d = np.load(os.path.join(GOLDEN, "int8_source_vectors.npz"))
    name, x, g, r0, c0 = SOURCE_CASES[i]
    src = DirectWeightSyncSource()
    try:
        src.register({"w": x.to(DEV)}, rank=0, tensor_slices={"w": source_quant_regimes.local_slice(x.shape, r0, c0)}, quantize={"w": g},
                     quant_dtype=I8)
        q, s, _ = src._quantized["w"]
        assert i8s.digest(q.view(torch.uint8).cpu().numpy()) == str(d[f"q_sha{i}"]), name
        assert i8.same_scales(s.cpu().numpy().reshape(d[f"s{i}"].shape), d[f"s{i}"]), name
        i8s.assert_exact(q, s, x, g, r0, c0)
    finally:
        run(src.cleanup())


def dequant_pull(q, s, g, r0, c0, dtype):
    """An int8 handle q (scale s) at global (r0, c0) pulled whole into a guarded `dtype` destination -> y."""
    src = DirectWeightSyncSource()
    sl = source_quant_regimes.local_slice(tuple(q.shape), r0, c0)
    try:
        h = src.register({"w": q.to(DEV)}, rank=0, tensor_slices={"w": sl}, **{KW[g]: {"w": s.to(DEV)}})["w"]
        base, y = guarded(tuple(q.shape), dtype)
        sync = DirectWeightSyncDest()
        run(sync.pull({"w": [h]}, {"w": y}, {"w": sl}))
        assert sync._int8_dequant_plans and not sync._dequant_plans
        sync.close()
        assert guards_intact(base)
    finally:
        run(src.cleanup())
    return y


DQ_CASES = i8s.dequant_inputs()


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("i", range(len(DQ_CASES)), ids=lambda i: DQ_CASES[i][0])
def test_int8_source_fixture_dequantised(i, dtype):
    d = np.load(os.path.join(GOLDEN, "int8_source_vectors.npz"))
    name, g, r0, c0, q, s = DQ_CASES[i]
    y = dequant_pull(q, s, g, r0, c0, dtype)
    # the fixture pins the numpy oracle's bits; the device matches them up to the NaN bit patterns (the platform's)
    ref = i8s.dequantize(q.numpy(), s.numpy(), g, r0, c0, str(dtype)[6:])
    assert i8s.digest(ref) == str(d[f"dq_{str(dtype)[6:]}_sha{i}"]), name
    got, nan = i8s.bits_of(y.cpu()), torch.isnan(y.float()).cpu().numpy()
    assert np.array_equal(got[~nan], ref[~nan]), name
    want = i8s.torch_dequantize(q.to(DEV), s.to(DEV), g, r0, c0, dtype)
    assert torch.equal(y.view(torch.uint8), want.view(torch.uint8)), name


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
def test_every_byte_against_the_scale_set(dtype):
    """All 256 int8 values times 1, a power of two, amax/127, f32-subnormal products, f16 / bf16 overflow, 0, a
    negative scale, Inf and NaN: torch CUDA bit for bit (NaN bytes included), the numpy oracle NaN-agnostically."""
    q = torch.arange(-128, 128, dtype=torch.int16).to(I8).repeat(len(i8s.SCALE_SET), 1)
    s = torch.from_numpy(i8s.SCALE_SET.copy()).reshape(-1, 1)
    y = dequant_pull(q, s, "channel", 0, 0, dtype)
    want = i8s.torch_dequantize(q.to(DEV), s.to(DEV), "channel", 0, 0, dtype)
    assert torch.equal(y.view(torch.uint8), want.view(torch.uint8))
    got, ref = i8s.bits_of(y.cpu()), i8s.dequantize(q.numpy(), s.numpy(), "channel", 0, 0, str(dtype)[6:])
    nan = torch.isnan(y.float()).cpu().numpy()
    assert np.array_equal(got[~nan], ref[~nan])
    if dtype == torch.float32:  # the subnormal products are there and kept
        tiny = (y.abs() < torch.finfo(torch.float32).tiny) & (y != 0)
        assert int(tiny.sum()) > 0


# ---- past byte 2^32 ----------------------------------------------------------------------------------
BIG = (129, 4096, 8192)


def big_bf16(seed):
    gen = torch.Generator(DEV).manual_seed(seed)
    x = torch.empty(BIG, dtype=torch.bfloat16, device=DEV)
    for e in range(BIG[0]):
        x[e] = torch.randn(BIG[1:], device=DEV, generator=gen) * (0.01 * (1 + e % 5))
    return x


def test_int8_quantising_pull_past_byte_2_32():
    """A bf16 stack of 129 experts [4096, 8192]: its source (8.7 GB) and each int8 destination (4.3 GB) run past
    byte 2^32; block, channel and tensor scales in turn, experts 0, 127 and 128 against torch CUDA."""
    n = int(np.prod(BIG))
    assert n > 2**32
    skip_unless_free(3 * n)
    x = big_bf16(16)
    src = DirectWeightSyncSource()
    try:
        h = src.register({"w": x}, rank=0)["w"]
        for g in i8.GRANULARITIES:
            qb, q = guarded(BIG, I8)
            sb, s = guarded(dest_scale_shape(g, BIG), torch.float32)
            sync = DirectWeightSyncDest()
            run(sync.pull({"w": [h]}, {"w": q}, **{KW[g]: {"w": s}}))
            for e in (0, 127, 128):
                want_q, want_s = i8.torch_quantize(x[e], g)
                assert torch.equal(q[e], want_q), (g, e)
                assert torch.equal(s[e].reshape(-1).view(torch.int32), want_s.reshape(-1).view(torch.int32)), (g, e)
            assert guards_intact(qb) and guards_intact(sb), g
            sync.close()
            del q, s, qb, sb, sync
            torch.cuda.empty_cache()
    finally:
        run(src.cleanup())
        del x
        torch.cuda.empty_cache()


def test_int8_staging_past_byte_2_32():
    """The same stack quantised on the source into int8 staging (4.3 GB) at each granularity; experts 0, 127 and 128
    against torch CUDA."""
    n = int(np.prod(BIG))
    skip_unless_free(3 * n + 2**30)
    x = big_bf16(15)
    try:
        for g in i8.GRANULARITIES:
            src = DirectWeightSyncSource()
            src.register({"w": x}, rank=0, quantize={"w": g}, quant_dtype=I8)
            q, s, _ = src._quantized["w"]
            for e in (0, 127, 128):
                want_q, want_s = i8s.torch_quantize(x[e], g)
                assert torch.equal(q[e], want_q), (g, e)
                assert torch.equal(s[e].reshape(-1).view(torch.int32), want_s.reshape(-1).view(torch.int32)), (g, e)
            run(src.cleanup())
            del q, s, src
            torch.cuda.empty_cache()
    finally:
        del x
        torch.cuda.empty_cache()


def test_int8_dequantising_pull_past_byte_2_32():
    """A channel-scaled int8 stack of 129 experts [4096, 8192] (4.3 GB) into bf16 (8.7 GB): the source shard and the
    destination both run past byte 2^32; experts 0, 127 and 128 against the torch CUDA rendering."""
    n = int(np.prod(BIG))
    skip_unless_free(3 * n)
    gen = torch.Generator(DEV).manual_seed(17)
    q = torch.empty(BIG, dtype=I8, device=DEV)
    for e in range(BIG[0]):
        q[e] = torch.randint(-128, 128, BIG[1:], dtype=I8, device=DEV, generator=gen)
    s = global_scale("channel", BIG, 17).to(DEV)
    sources, handles = register_boxes(q, [whole(BIG)], granularity="channel",
                                      scale_of=partial(dq_local_scale, s, "channel"))
    sync, y, _, (base,) = pull_box(handles, BIG, whole(BIG), torch.bfloat16)
    try:
        assert sync._int8_dequant_plans
        for e in (0, 127, 128):
            assert torch.equal(y[e], i8s.torch_dequantize(q[e], s[e], "channel")), e
        assert guards_intact(base)
    finally:
        sync.close()
        cleanup(sources)
        del q, y, base, sources, handles
        torch.cuda.empty_cache()


# ---- random layouts ----------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(24, 48))
def test_random_layouts_with_special_values(seed):
    quant_pull_regimes.run_random_layout(seed, dst_dtype=I8)


@pytest.mark.parametrize("seed", range(24))
def test_random_dequant_layouts_from_int8_handles(seed):
    w = fp8_regimes.draw(random.Random(9800 + seed), "dequant", seed)
    q, s = fp8_regimes.inputs(w, "finite", I8)
    sources, handles = register_boxes(q, list(w.src), granularity=w.sg, scale_of=partial(dq_local_scale, s, w.sg))
    sync, y, _, (base,) = pull_box(handles, w.shape, w.dst, fp8_regimes.DST[w.out])
    try:
        with named(f"seed {seed}: {w.describe()}"):
            fp8_regimes.live_tables(sync, y, int8_src=True)
            fp8_regimes.assert_int8_dequantised(y, q, s, w.sg, w.dst)
            assert guards_intact(base)
    finally:
        sync.close()
        cleanup(sources)

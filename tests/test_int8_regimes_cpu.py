"""INT8 in every workload of the three regime catalogues, and the int8 rounding-edge generator, without a GPU.

* The quantising pulls (tests/quant_pull_regimes.py) into int8 destinations (TSB_I8 rects), source-side quantisation
  (tests/source_quant_regimes.py) into int8 staging (``dst_dtype=TSB_I8``) and the dequantising pulls (the ``dq_*``
  workloads of tests/fp8_regimes.py) from int8 handles (TSB_I8 source rects), each compiled on host memory: the
  tables are byte for byte the float8_e4m3fn ones from the same buffers, every regime still holds on them, and
  replayed with the int8 interpreters they give the numpy oracles and the torch CPU rendering bit for bit.
* The edge generator of oracle/int8_oracle.py checked in numpy: the renderings on known inputs, every planted value
  telling the formula from the wrong rendering it is planted for, and every route shape reaching all of them."""

import contextlib
import functools
from unittest import mock

import numpy as np
import pytest
import torch

from oracle import int8_oracle as i8
from oracle import int8_source_oracle as i8s
from oracle.ue8m0_oracle import group_amax, group_ids
from tests import fp8_regimes, quant_pull_regimes, source_quant_regimes
from tests import test_dequant_fp8_cpu as dq_cpu
from tests import test_requant_fp8_cpu as rq_cpu
from tests.helpers import dest_scale_shape, region
from tests.test_quant_pull_regimes_cpu import host_shard, workload_inputs
from tests.test_source_quant_cpu import host_shard as source_shard
from tests.test_source_quant_regimes_cpu import workload_inputs as source_inputs
from torchstore_b200 import _native
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, RDMAWeightHandle
from torchstore_b200.planner import StridedMem
from torchstore_b200.transport.types import TensorSlice

DQ_WORKLOADS = sorted(n for n, w in fp8_regimes.WORKLOADS.items() if w.kind == "dequant")
DQ_REGIMES = sorted(n for n, r in fp8_regimes.REGIMES.items() if fp8_regimes.WORKLOADS[r.workload].kind == "dequant")


def same_tables(a, b, what):
    assert len(a) == len(b), what
    for x, y in zip(a, b):
        assert (x.dtype == y.dtype and x.tobytes() == y.tobytes()) if isinstance(x, np.ndarray) else x == y, what


@contextlib.contextmanager
def fp8_compared(field):
    """Every block / scaled / dequantising *_compile_host call is given TSB_I8 rects (on the rects' `field` side) and
    compiles again from the same buffers with them relabelled TSB_F8E4M3; the tables must be byte-identical."""
    seen = []

    def wrap(kind, orig):
        def compile_(device, rects, n, *rest):
            assert n and all(getattr(rects[i], field) == _native.TSB_I8 for i in range(n)), kind
            got = orig(device, rects, n, *rest)
            for i in range(n):
                setattr(rects[i], field, _native.TSB_F8E4M3)
            try:
                plain = orig(device, rects, n, *rest)
            finally:
                for i in range(n):
                    setattr(rects[i], field, _native.TSB_I8)
            same_tables(got if isinstance(got, tuple) else (got,), plain if isinstance(plain, tuple) else (plain,), kind)
            seen.append(kind)
            return got
        return compile_

    kinds = ("block_fp8", "scaled_fp8") if field == "dst_dtype" else ("dequant_fp8",)
    with contextlib.ExitStack() as stack:
        for kind in kinds:
            name = f"{kind}_compile_host"
            stack.enter_context(mock.patch.object(_native, name, wrap(kind, getattr(_native, name))))
        yield seen


def assert_torch_cpu(q, s, want_q, want_s):
    assert np.array_equal(q, want_q.numpy())
    assert i8.same_scales(np.asarray(s).reshape(-1), want_s.numpy().reshape(-1))


# ---- quantising pulls into int8 ----------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def quant_pull(name):
    """Plan workload `name` on host memory into int8 destinations, replay it -> (tables, geometry, xs, dests, scales)."""
    w = quant_pull_regimes.WORKLOADS[name]
    xs = workload_inputs(name)
    handles, dests, scales, slices = {}, {}, {}, {}
    for i, (p, x) in enumerate(zip(w.pulls, xs)):
        n = f"w{i}"
        handles[n] = [RDMAWeightHandle(rdma_buffer=host_shard(x, off, loc, p.shift(r)),
                                       tensor_slice=TensorSlice(off, (r,), p.shape, loc, (len(p.src),)), source_rank=r)
                      for r, (off, loc) in enumerate(p.src)]
        off, loc = p.dst
        dests[n] = torch.full(loc, 0x55, dtype=torch.int8)
        scales[n] = torch.full(dest_scale_shape(p.g, loc), -1.0)
        slices[n] = TensorSlice(off, (0,), p.shape, loc, (1,))
    ops = DirectWeightSyncDest()._build_plan(handles, dests, slices)
    with fp8_compared("dst_dtype") as seen:
        tables, geom = quant_pull_regimes.compile_tables(w.pulls, ops, handles, StridedMem.from_tensor, dests, scales)
    assert seen
    if tables.block is not None:
        i8.replay_block(*tables.block)
    if tables.scaled is not None:
        i8.replay_scaled(*tables.scaled)
    return tables, geom, xs, dests, scales, handles


@pytest.mark.parametrize("name", sorted(quant_pull_regimes.WORKLOADS))
def test_quant_pull_workload_replays_to_the_int8_oracle(name):
    _, _, xs, dests, scales, _ = quant_pull(name)
    for i, (p, x) in enumerate(zip(quant_pull_regimes.WORKLOADS[name].pulls, xs)):
        xr = region(x, *p.dst)
        q, s = dests[f"w{i}"].numpy(), scales[f"w{i}"].numpy()
        xf = i8.widen(i8.bits_of(xr), p.dtype)
        want_q, want_s = i8.quantize(xf, p.g)
        assert np.array_equal(q, want_q), p.describe()
        assert np.array_equal(s.reshape(-1).view(np.uint32), want_s.reshape(-1).view(np.uint32)), p.describe()
        assert_torch_cpu(q, s, *i8.torch_quantize(xr, p.g))
        i8s.assert_invariants(q, xf, p.g)


@pytest.mark.parametrize("regime", sorted(quant_pull_regimes.REGIMES))
def test_quant_pull_regime_holds_on_the_int8_tables(regime):
    r = quant_pull_regimes.REGIMES[regime]
    tables, geom, *_ = quant_pull(r.workload)
    assert r.holds(tables, geom), regime


# ---- source-side int8 staging ------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def source_quant(name):
    w = source_quant_regimes.WORKLOADS[name]
    keep, targets = [], []
    for t, x in zip(w.targets, source_inputs(name)):
        backing, q, s, tgt = source_shard(x, t.granularity, t.row0, t.col0, t.misalign)
        keep.append((x, q, s, backing))
        targets.append(tgt)
    arr = _native.make_source_quant_target_array(len(targets))
    for i, t in enumerate(targets):
        arr[i] = t
    tables = _native.source_quant_compile_host(0, arr, len(targets), dst_dtype=_native.TSB_I8)
    same_tables(tables, _native.source_quant_compile_host(0, arr, len(targets), dst_dtype=_native.TSB_F8E4M3), name)
    i8s.replay_source(*tables)
    return tables, [_native.SourceQuantTarget.from_buffer_copy(t) for t in targets], keep


@pytest.mark.parametrize("name", sorted(source_quant_regimes.WORKLOADS))
def test_source_workload_replays_to_the_int8_oracle(name):
    _, _, keep = source_quant(name)
    for t, (x, q, s, _) in zip(source_quant_regimes.WORKLOADS[name].targets, keep):
        q = q.view(np.int8)
        xf = i8.widen(i8.bits_of(x), t.dtype)
        want_q, want_s = i8s.quantize(xf, t.granularity, t.row0, t.col0)
        assert np.array_equal(q, want_q), t.describe()
        assert np.array_equal(s.view(np.uint32), want_s.view(np.uint32)), t.describe()
        assert_torch_cpu(q, s, *i8s.torch_quantize(x, t.granularity, t.row0, t.col0))
        i8s.assert_invariants(q, xf, t.granularity, t.row0, t.col0)


@pytest.mark.parametrize("regime", sorted(source_quant_regimes.REGIMES))
def test_source_regime_holds_on_the_int8_tables(regime):
    r = source_quant_regimes.REGIMES[regime]
    tables, targets, _ = source_quant(r.workload)
    assert r.holds(tables, targets), regime


# ---- dequantising pulls from int8 handles ------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def dequant(name):
    w = fp8_regimes.WORKLOADS[name]
    q, s = i8s.int8_of(w.shape, w.seed), rq_cpu.global_scale(w.sg, w.shape, w.seed)
    with fp8_compared("src_dtype") as seen:
        dest, tiles, (_, _, arr, _) = dq_cpu.compile_pull(q, s, w.sg, list(w.src), w.dst, getattr(torch, w.out))
    assert seen == ["dequant_fp8"]
    i8s.replay_dequant(tiles)
    geom = fp8_regimes.geometry(dest.data_ptr(), w.dst[1], fp8_regimes.ES[w.out], arr, len(arr))
    return q, s, dest, tiles, geom


@pytest.mark.parametrize("name", DQ_WORKLOADS)
def test_dequant_workload_replays_to_the_int8_oracle(name):
    w = fp8_regimes.WORKLOADS[name]
    q, s, dest, _, _ = dequant(name)
    off, loc = w.dst
    qr, sr = region(q, off, loc), dq_cpu.local_scale(s, w.sg, off, loc)
    want = i8s.dequantize(qr.numpy(), sr.numpy(), w.sg, off[-2], off[-1], w.out)
    assert np.array_equal(i8s.bits_of(dest), want), w.describe()
    torch_want = i8s.torch_dequantize(qr, sr, w.sg, off[-2], off[-1], getattr(torch, w.out))
    assert torch.equal(dest.view(torch.uint8), torch_want.view(torch.uint8)), w.describe()


@pytest.mark.parametrize("regime", DQ_REGIMES)
def test_dequant_regime_holds_on_the_int8_tables(regime):
    r = fp8_regimes.REGIMES[regime]
    *_, tiles, geom = dequant(r.workload)
    assert r.holds(tiles, geom), regime


# ---- the edge generator ------------------------------------------------------------------------------
def test_renderings_on_known_inputs():
    x = np.array([2.5, -2.5, 3.5, 2.7, -2.7, 0.49], dtype=np.float32)
    assert i8.render("formula", x, 1, 1).tolist() == [2, -2, 4, 3, -3, 0]
    assert i8.render("half_away_from_zero", x, 1, 1).tolist() == [3, -3, 4, 3, -3, 0]
    assert i8.render("truncation", x, 1, 1).tolist() == [2, -2, 3, 2, -2, 0]
    for name in i8.RENDERINGS:  # NaN -> 0 and saturation in every rendering
        assert i8.render(name, np.array([np.nan, 1e9, -1e9], np.float32), 1, 1).tolist() == [0, 127, -128]
    # scale exactly 1 (amax 127): the scale-side slips agree with the formula
    v = np.linspace(-127, 127, 10001).astype(np.float32)
    assert not any(m.any() for n, m in i8.discriminated(v, 127).items() if n in i8.HARD)


@pytest.mark.parametrize("dtype", ("bfloat16", "float16", "float32"))
def test_clamp_amaxes_straddle_the_floor(dtype):
    a = i8.clamp_amaxes(dtype)
    floor = np.float32(1e-4)
    assert a[0] < a[1] < a[2] and a[0] < floor < a[2] and (a[1] == floor if dtype == "float32" else a[1] < floor)
    held = i8.widen(i8.bits_of(torch.from_numpy(a).to(getattr(torch, dtype))), dtype)
    assert np.array_equal(held.view(np.uint32), a.view(np.uint32))  # each is a value of the dtype


@pytest.mark.parametrize("dtype", ("bfloat16", "float16", "float32"))
def test_every_edge_value_tells_a_rendering_apart(dtype):
    groups = i8.edge_groups(dtype)
    assert len(groups) == 16 and [float(a) for a, _ in groups[:4]] == [float(v) for v in i8.clamp_amaxes(dtype)] + [127.0]
    counts = dict.fromkeys(i8.HARD, 0)
    for a, vals in groups:
        assert len(vals) and (vals > 0).all() and (vals <= a).all()
        held = i8.widen(i8.bits_of(torch.from_numpy(vals).to(getattr(torch, dtype))), dtype)
        assert np.array_equal(held.view(np.uint32), vals.view(np.uint32))
        told = i8.discriminated(vals, a)
        assert np.any(list(told.values()), axis=0).all()  # each value differs from the formula somewhere
        for h in i8.HARD:
            counts[h] += int(told[h].any())
    assert min(counts.values()) >= 2, counts


ROUTE_SHAPES = {"block": (128, 128 * 16), "channel": (16, 160), "tensor": (16, 16, 64)}


@pytest.mark.parametrize("dtype", (torch.bfloat16, torch.float16, torch.float32), ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("g", sorted(ROUTE_SHAPES))
def test_planted_values_tell_their_renderings_apart(g, dtype):
    for r0, c0 in ((0, 0), (37, 70)):
        x, n = i8.plant_rounding_edges(ROUTE_SHAPES[g], dtype, g, r0, c0)
        told, ties = i8.told_apart(x, g, r0, c0)
        assert told == set(i8.WRONG) and len(ties) == 4, (told, ties)
        xf = i8.widen(i8.bits_of(x), str(dtype)[6:])
        gid, ng = group_ids(g, tuple(x.shape), r0, c0)
        amax = group_amax(xf, gid, ng)[gid]
        hit = np.any(list(i8.discriminated(xf, amax).values()), axis=0)
        planted = (np.abs(xf) != amax) & (xf != 0)
        assert hit[planted].all()  # every value but the amax elements differs from the formula in some rendering

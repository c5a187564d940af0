"""Power-of-two (UE8M0) scales in every workload of the three regime catalogues, without a GPU.

* The quantising pulls (tests/quant_pull_regimes.py), source-side quantisation (tests/source_quant_regimes.py) and
  the requantising pulls (the ``rq_*`` workloads of tests/fp8_regimes.py), each compiled on host memory with
  ``TSB_QUANT_UE8M0``: the tables are byte for byte the ones flags 0 gives from the same buffers, every regime still
  holds on them, and replayed with ``scale_fmt="ue8m0"`` they give the numpy UE8M0 oracle bit for bit and the torch
  CPU rendering (NaN-agnostic inside non-finite groups).
* The lossless-requantise property on every requantising workload whose destination groups each lie inside one
  source group, with the source scales replaced by powers of two in [2^-22, 2^119]."""

import contextlib
import functools
from unittest import mock

import numpy as np
import pytest
import torch

from oracle import ue8m0_oracle as u8
from oracle.dequant_fp8_oracle import decode_e4m3, expand
from tests import fp8_regimes, quant_pull_regimes, source_quant_regimes
from tests import test_fp8_regimes_cpu as fp8_cpu
from tests import test_requant_fp8_cpu as rq_cpu
from tests.helpers import region
from tests.test_quant_pull_regimes_cpu import compiled
from tests.test_source_quant_cpu import compile_host, host_shard
from tests.test_source_quant_regimes_cpu import workload_inputs as source_inputs
from torchstore_b200 import _native

UE8M0 = _native.TSB_QUANT_UE8M0
KINDS = ("block_fp8", "scaled_fp8", "source_quant", "requant_fp8")
RQ_WORKLOADS = sorted(n for n, w in fp8_regimes.WORKLOADS.items() if w.kind == "requant")
RQ_REGIMES = sorted(n for n, r in fp8_regimes.REGIMES.items() if fp8_regimes.WORKLOADS[r.workload].kind == "requant")


def u32(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


@contextlib.contextmanager
def flags_compared():
    """Every quantising *_compile_host call also compiles with flags 0 from the same buffers; the tables must be
    byte-identical.  Yields the list of kinds compiled."""
    seen = []

    def wrap(kind, orig):
        def compile_(*args):
            got, plain = orig(*args), orig(*args[:-1], 0)
            assert args[-1] == UE8M0 and len(got) == len(plain), kind
            for a, b in zip(got, plain):
                assert (a.dtype == b.dtype and a.tobytes() == b.tobytes()) if isinstance(a, np.ndarray) else a == b, kind
            seen.append(kind)
            return got
        return compile_

    with contextlib.ExitStack() as stack:
        for kind in KINDS:
            name = f"{kind}_compile_host"
            stack.enter_context(mock.patch.object(_native, name, wrap(kind, getattr(_native, name))))
        yield seen


def assert_torch_cpu(q, s, want_q, want_s):
    """q, s (numpy) against the torch CPU rendering: bit-exact, NaN-agnostic inside non-finite groups."""
    want_q, want_s = want_q.view(torch.uint8).numpy(), want_s.numpy().reshape(s.shape)
    nan_w = (want_q & 0x7F) == 0x7F
    assert np.array_equal((q & 0x7F) == 0x7F, nan_w) and np.array_equal(q[~nan_w], want_q[~nan_w])
    assert np.array_equal(np.isnan(s), np.isnan(want_s))
    assert np.array_equal(u32(s)[~np.isnan(s)], u32(want_s)[~np.isnan(want_s)])


# ---- quantising pulls --------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def quant_pull(name):
    with flags_compared() as seen:
        tables, geom, xs, dests, scales, _ = compiled(name, UE8M0)
    assert seen
    if tables.block is not None:
        u8.replay_block(*tables.block, scale_fmt="ue8m0")
    if tables.scaled is not None:
        u8.replay_scaled(*tables.scaled, scale_fmt="ue8m0")
    return tables, geom, xs, dests, scales


@pytest.mark.parametrize("name", sorted(quant_pull_regimes.WORKLOADS))
def test_quant_pull_workload_replays_to_the_ue8m0_oracle(name):
    _, _, xs, dests, scales = quant_pull(name)
    for i, (p, x) in enumerate(zip(quant_pull_regimes.WORKLOADS[name].pulls, xs)):
        xr = region(x, *p.dst)
        q, s = dests[f"w{i}"].view(torch.uint8).numpy(), scales[f"w{i}"].numpy()
        want_q, want_s = u8.quantize(xr.float().numpy(), p.g, scale_fmt="ue8m0")
        assert np.array_equal(q, want_q), p.describe()
        assert np.array_equal(u32(s).reshape(-1), u32(want_s).reshape(-1)), p.describe()
        assert_torch_cpu(q, s, *u8.torch_quantize(xr, p.g, scale_fmt="ue8m0"))


@pytest.mark.parametrize("regime", sorted(quant_pull_regimes.REGIMES))
def test_quant_pull_regime_holds_on_the_ue8m0_tables(regime):
    r = quant_pull_regimes.REGIMES[regime]
    tables, geom, *_ = quant_pull(r.workload)
    assert r.holds(tables, geom), regime


# ---- source-side quantisation ------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def source_quant(name):
    w = source_quant_regimes.WORKLOADS[name]
    keep, targets = [], []
    for t, x in zip(w.targets, source_inputs(name)):
        backing, q, s, tgt = host_shard(x, t.granularity, t.row0, t.col0, t.misalign)
        keep.append((x, q, s, backing))
        targets.append(tgt)
    with flags_compared() as seen:
        tables = compile_host(targets, UE8M0)
    assert seen == ["source_quant"]
    u8.replay_source(*tables, scale_fmt="ue8m0")
    return tables, [_native.SourceQuantTarget.from_buffer_copy(t) for t in targets], keep


@pytest.mark.parametrize("name", sorted(source_quant_regimes.WORKLOADS))
def test_source_workload_replays_to_the_ue8m0_oracle(name):
    _, _, keep = source_quant(name)
    for t, (x, q, s, _) in zip(source_quant_regimes.WORKLOADS[name].targets, keep):
        want_q, want_s = u8.quantize(u8.widen(u8.bits_of(x), t.dtype), t.granularity, t.row0, t.col0, scale_fmt="ue8m0")
        assert np.array_equal(q, want_q), t.describe()
        assert np.array_equal(u32(s), u32(want_s)), t.describe()
        assert_torch_cpu(q, s, *u8.torch_quantize(x, t.granularity, t.row0, t.col0, scale_fmt="ue8m0"))


@pytest.mark.parametrize("regime", sorted(source_quant_regimes.REGIMES))
def test_source_regime_holds_on_the_ue8m0_tables(regime):
    r = source_quant_regimes.REGIMES[regime]
    tables, targets, _ = source_quant(r.workload)
    assert r.holds(tables, targets), regime


# ---- requantising pulls ------------------------------------------------------------------------------
def requant(name, q, s):
    """Compile workload `name` over (q, s) with TSB_QUANT_UE8M0 and replay it -> (dest, dest_scale, tables, geom)."""
    w = fp8_regimes.WORKLOADS[name]
    with flags_compared() as seen:
        dest, dest_scale, tables, keep = rq_cpu.compile_pull(q, s, w.sg, list(w.src), w.dst, w.out, UE8M0)
    assert seen == ["requant_fp8"]
    geom = fp8_regimes.geometry(dest.data_ptr(), w.dst[1], 1, keep[2], len(keep[2]))
    u8.replay_requant(*tables, scale_fmt="ue8m0")
    return dest, dest_scale, tables, geom


@functools.lru_cache(maxsize=None)
def requant_catalogue(name):
    q, s = fp8_cpu.inputs(fp8_regimes.WORKLOADS[name])
    return (q, s) + requant(name, q, s)


@pytest.mark.parametrize("name", RQ_WORKLOADS)
def test_requant_workload_replays_to_the_ue8m0_oracle(name):
    w = fp8_regimes.WORKLOADS[name]
    q, s, dest, dest_scale, _, _ = requant_catalogue(name)
    off, loc = w.dst
    args = (region(q, off, loc), rq_cpu.local_scale(s, w.sg, off, loc), w.sg, off[-2], off[-1], w.out)
    want_q, want_s = u8.requantize(args[0].view(torch.uint8).numpy(), args[1].numpy(), *args[2:], scale_fmt="ue8m0")
    got_q, got_s = dest.view(torch.uint8).numpy(), dest_scale.numpy()
    assert np.array_equal(got_q, want_q), w.describe()
    assert np.array_equal(u32(got_s).reshape(-1), u32(want_s).reshape(-1)), w.describe()
    assert_torch_cpu(got_q, got_s, *u8.torch_requantize(*args, scale_fmt="ue8m0"))


@pytest.mark.parametrize("regime", RQ_REGIMES)
def test_requant_regime_holds_on_the_ue8m0_tables(regime):
    r = fp8_regimes.REGIMES[regime]
    *_, tables, geom = requant_catalogue(r.workload)
    assert r.holds(tables, geom), regime


# ---- the lossless-requantise domain ------------------------------------------------------------------
def contained(w) -> bool:
    """Every destination group of workload `w` lies inside one global source group."""
    off, loc = w.dst
    dst, n_dst = u8.group_ids(w.out, loc)
    src, _ = u8.group_ids(w.sg, tuple(o + e for o, e in zip(off, loc)))
    src = src[tuple(slice(o, None) for o in off)]
    pairs = np.unique(np.stack([dst.reshape(-1), src.reshape(-1)]), axis=1)
    return pairs.shape[1] == n_dst


# requantising workloads whose destination groups each lie inside one source group: coinciding groups, and the
# last 22-row block of rq_block_fsdp6_rows inside its 128-row source block
LOSSLESS = ["rq_band_narrow", "rq_band_tall", "rq_block_aligned", "rq_block_fsdp6_rows", "rq_block_moe",
            "rq_channel_long_channel_src", "rq_tensor_aligned_moe", "rq_tensor_long_rows", "rq_tensor_many_groups"]


def test_lossless_workloads_are_decided_by_geometry():
    assert sorted(n for n in RQ_WORKLOADS if contained(fp8_regimes.WORKLOADS[n])) == LOSSLESS


def assert_lossless(q, s, sg, y, ys, dg, off, loc):
    """f32(q') * s' == f32(q) * s element for element over the window, and s' <= s group by group."""
    qw = region(q, off, loc).view(torch.uint8).numpy()
    sw = rq_cpu.local_scale(s, sg, off, loc).numpy()
    before = decode_e4m3(qw) * expand(sw, loc, sg, off[-2], off[-1])
    after = decode_e4m3(y) * expand(np.asarray(ys, np.float32).reshape(rq_cpu.dest_scale_shape(dg, loc)), loc, dg)
    assert np.isfinite(before).all()
    assert np.array_equal(u32(after), u32(before))
    assert (expand(np.asarray(ys, np.float32).reshape(rq_cpu.dest_scale_shape(dg, loc)), loc, dg)
            <= expand(sw, loc, sg, off[-2], off[-1])).all()


@pytest.mark.parametrize("name", LOSSLESS)
def test_lossless_requantise_by_replay(name):
    w = fp8_regimes.WORKLOADS[name]
    q, s = fp8_cpu.inputs(w)
    s = torch.from_numpy(u8.pow2_scales(tuple(s.shape), w.seed))
    dest, dest_scale, _, _ = requant(name, q, s)
    assert_lossless(q, s, w.sg, dest.view(torch.uint8).numpy(), dest_scale.numpy(), w.out, *w.dst)

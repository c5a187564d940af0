"""Power-of-two (UE8M0) scales on the H100 in the regimes the float32 suites reach, at the scale step's edges in
every route, over the torch CPU fixture and over the lossless-requantise domain.

* Regimes: every regime of tests/quant_pull_regimes.py, tests/source_quant_regimes.py and the ``rq_*`` regimes of
  tests/fp8_regimes.py, in each catalogue's own variants, with ``scale_fmt="ue8m0"``: the regime re-asserted from
  the live plan's tables, bit-exact with the torch CUDA rendering (NaN bytes and scale_inv included) and with the
  numpy oracle on finite groups, guard bytes intact, and every finite scale_inv a power of two in [t, 2t) of the
  float32 formula's t for the same group.
* Edges: every value of ``edge_amaxes()`` (and its bf16 / f16 counterparts) the amax of its own group, beside an
  all-zero and an all-subnormal group, in every quantising, source-side and requantising route; each route reaches
  the step's three branches (keep, round up, clamp), decided from the inputs.
* The fixture tests/golden/ue8m0_vectors.npz on the device, as pulls at (0, 0) and as source shards at (37, 70).
* Lossless requantising: power-of-two source scales in [2^-22, 2^119] keep every value when each destination group
  lies inside one source group (coinciding or contained), and the ends of that domain pinned: the read-back
  overflow at amax >= 248 * 2^120, and source scales under 2^-22.
* One state-dict round trip with ``quantize=`` and ``scale_fmt="ue8m0"``."""

from functools import partial

import numpy as np
import pytest
import torch

import torchstore_b200 as ts
from oracle import ue8m0_oracle as u8
from oracle.dequant_fp8_oracle import decode_e4m3, expand, torch_dequantize
from tests import fp8_regimes, quant_pull_regimes, source_quant_regimes
from tests import test_fp8_regimes_cpu as fp8_cpu
from tests.helpers import (DEV, E4M3, KW, cleanup, dest_scale_shape, guarded, guards_intact, named, native_session,
                           pull_box, region, register_boxes, run)
from tests.quant_pull_regimes import Pull
from tests.source_quant_regimes import assert_exact
from tests.test_dequant_fp8_cpu import local_scale as dq_local_scale
from tests.test_ue8m0_cpu import fixture_cases, is_pow2, u32
from tests.test_ue8m0_regimes_cpu import LOSSLESS, RQ_REGIMES, assert_lossless
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource

pytestmark = pytest.mark.gpu
UE = "ue8m0"
DTYPES = (torch.bfloat16, torch.float16, torch.float32)
_init = pytest.fixture(scope="module", autouse=True)(native_session)


def whole(shape):
    return ((0,) * len(shape), tuple(shape))


# ---- every regime in UE8M0 ---------------------------------------------------------------------------
@pytest.mark.parametrize("variant", quant_pull_regimes.VARIANTS)
@pytest.mark.parametrize("regime", sorted(quant_pull_regimes.REGIMES))
def test_quant_pull_regime(regime, variant):
    quant_pull_regimes.run_regime(regime, variant, UE)


@pytest.mark.parametrize("variant", source_quant_regimes.VARIANTS)
@pytest.mark.parametrize("regime", sorted(source_quant_regimes.REGIMES))
def test_source_regime(regime, variant):
    source_quant_regimes.run_regime(regime, variant, UE)


@pytest.mark.parametrize("name", sorted(source_quant_regimes.WORKLOADS))
def test_source_workload_writes_nothing_outside_its_outputs(name):
    source_quant_regimes.run_guarded(name, UE)


@pytest.mark.parametrize("variant", fp8_regimes.VARIANTS)
@pytest.mark.parametrize("regime", RQ_REGIMES)
def test_requant_regime(regime, variant):
    fp8_regimes.run_regime(regime, variant, UE)


# ---- the step's edges, route by route ----------------------------------------------------------------
def n_edge_groups(dtype) -> int:
    return len(u8.edge_amaxes_for(dtype)) + 3  # the edges, a zero group, a subnormal group, one random group


def assert_all_branches(branches):
    assert set(u8.BRANCHES) <= set(branches.tolist()), sorted(set(branches.tolist()))


QUANT_ROUTES = {  # route -> (granularity, shape of G groups, kind of the pass the plan must hold)
    "block_kernel": ("block", lambda G: (128, 128 * G), "block"),
    "rows_kernel": ("channel", lambda G: (G, 160), "bands"),
    "tensor_two_pass": ("tensor", lambda G: (G, 16, 64), "tiles"),
    "long_row_channel_two_pass": ("channel", lambda G: (G, 16400), "tiles"),
}


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("route", sorted(QUANT_ROUTES))
def test_edges_of_a_quantising_pull(route, dtype):
    g, shape_of, kind = QUANT_ROUTES[route]
    shape = shape_of(n_edge_groups(dtype))
    if route == "long_row_channel_two_pass" and dtype == torch.float32:
        shape = (shape[0], 8200)  # over the 32 KiB row stage
    x, branches = u8.plant_edges(shape, dtype, g, seed=len(route))
    assert_all_branches(branches)
    name = str(dtype)[6:]
    p = Pull(name, shape, quant_pull_regimes.split(shape, 2, -1), whole(shape), g)
    pulled = quant_pull_regimes.Pulled((p,), [x], scale_fmt=UE)
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


SOURCE_ROUTES = {  # route -> (granularity, shard shape of at least G groups at (37, 70))
    "block_units": ("block", lambda G: (300, 128 * (G // 3 + 1))),
    "channel_units": ("channel", lambda G: (G, 200)),
    "tensor_tiles": ("tensor", lambda G: (G, 16, 64)),
}


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("route", sorted(SOURCE_ROUTES))
def test_edges_of_source_side_quantisation(route, dtype):
    g, shape_of = SOURCE_ROUTES[route]
    shape = shape_of(n_edge_groups(dtype))
    x, branches = u8.plant_edges(shape, dtype, g, 37, 70, seed=len(route))
    assert_all_branches(branches)
    src = DirectWeightSyncSource()
    try:
        src.register({"w": x.to(DEV)}, rank=0, tensor_slices={"w": source_quant_regimes.local_slice(shape, 37, 70)}, quantize={"w": g},
                     scale_fmt=UE)
        q, s, _ = src._quantized["w"]
        with named(f"{route} {str(dtype)[6:]}"):
            assert_exact(q, s, x, g, 37, 70, UE)
    finally:
        run(src.cleanup())


REQUANT_ROUTES = {  # route -> (granularity of both sides, layout of the G groups)
    "staged_block": "block",
    "staged_channel": "channel",
    "tensor_tiles": "tensor",
}


def edge_source(g: str):
    """A `g`-scaled fp8 tensor whose groups carry plant_edge_sources' groups -> (q, scale, branches)."""
    n = len(u8.edge_amaxes()) + 3
    group = {"block": (128, 128), "channel": (160,), "tensor": (16, 64)}[g]
    q, s = u8.plant_edge_sources(n, group, seed=n)
    if g == "block":
        q, s = q.transpose(1, 0, 2).reshape(128, 128 * n), s.reshape(1, n)
    elif g == "channel":
        s = s.reshape(n, 1)
    with np.errstate(all="ignore"):
        x = decode_e4m3(q) * expand(s, q.shape, g)
    gid, ng = u8.group_ids(g, q.shape)
    branches = u8.branch_of_amax(u8.group_amax(x.astype(np.float32), gid, ng))
    return torch.from_numpy(np.ascontiguousarray(q)).view(E4M3), torch.from_numpy(np.ascontiguousarray(s)), branches


@pytest.mark.parametrize("route", sorted(REQUANT_ROUTES))
def test_edges_of_a_requantising_pull(route):
    g = REQUANT_ROUTES[route]
    q, s, branches = edge_source(g)
    assert_all_branches(branches)
    box = whole(tuple(q.shape))
    sources, handles = register_boxes(q, [box], granularity=g, scale_of=partial(dq_local_scale, s, g))
    sync, y, ys, bases = pull_box(handles, tuple(q.shape), box, E4M3, granularity=g, requantize=True, scale_fmt=UE)
    try:
        tables, _ = fp8_regimes.live_tables(sync, y, ys, g)
        units, _, tiles, _ = tables
        assert (len(tiles) > 0) == (g == "tensor") and (len(units) > 0) == (g != "tensor")
        with named(route):
            fp8_regimes.assert_requant_oracle(y, ys, q, s, g, box, g, UE)
            fp8_regimes.assert_requant_torch_cuda(y, ys, q, s, g, box, g, UE)
        assert all(guards_intact(b) for b in bases)
    finally:
        sync.close()
        cleanup(sources)


# ---- the torch CPU fixture on the device -------------------------------------------------------------
INPUTS = {name: x for name, x, *_ in u8.fixture_inputs()}


def assert_fixture(q, s, want_q, want_s):
    s = s.reshape(want_s.shape)
    assert np.array_equal(np.isnan(s), np.isnan(want_s))
    fin = ~np.isnan(want_s)
    assert np.array_equal(u32(s)[fin], u32(want_s)[fin]) and is_pow2(s[np.isfinite(s)]).all()
    if isinstance(want_q, str):
        assert u8.digest(q) == want_q
    else:
        nan_q, nan_w = (q & 0x7F) == 0x7F, (want_q & 0x7F) == 0x7F
        assert np.array_equal(nan_q, nan_w) and np.array_equal(q[~nan_w], want_q[~nan_w])


@pytest.mark.parametrize("case", fixture_cases(), ids=lambda c: c[0])
def test_fixture_on_the_h100(case):
    name, _, g, r0, c0, want_q, want_s = case
    x = INPUTS[name]
    src = DirectWeightSyncSource()
    try:
        if (r0, c0) == (0, 0):
            h = src.register({"w": x.to(DEV)}, rank=0)["w"]
            qb, q = guarded(tuple(x.shape), E4M3)
            sb, s = guarded(dest_scale_shape(g, tuple(x.shape)), torch.float32)
            sync = DirectWeightSyncDest()
            run(sync.pull({"w": [h]}, {"w": q}, **{KW[g]: {"w": s}}, scale_fmt=UE))
            sync.close()
            assert guards_intact(qb) and guards_intact(sb)
        else:
            src.register({"w": x.to(DEV)}, rank=0, tensor_slices={"w": source_quant_regimes.local_slice(x.shape, r0, c0)}, quantize={"w": g},
                         scale_fmt=UE)
            q, s, _ = src._quantized["w"]
        assert_fixture(q.view(torch.uint8).cpu().numpy(), s.cpu().numpy(), want_q, want_s)
    finally:
        run(src.cleanup())


def test_fixture_runs_both_ways():
    where = {(c[3], c[4]) for c in fixture_cases()}
    assert where == {(0, 0), (37, 70)}


# ---- the lossless-requantise domain ------------------------------------------------------------------
@pytest.mark.parametrize("name", LOSSLESS)
def test_lossless_requantise_of_a_catalogue_workload(name):
    """Power-of-two source scales in [2^-22, 2^119], destination groups inside source groups: values kept."""
    w = fp8_regimes.WORKLOADS[name]
    q, s = fp8_cpu.inputs(w)
    s = torch.from_numpy(u8.pow2_scales(tuple(s.shape), w.seed))
    sources, handles = register_boxes(q, list(w.src), granularity=w.sg, scale_of=partial(dq_local_scale, s, w.sg))
    sync, y, ys, bases = pull_box(handles, w.shape, w.dst, E4M3, granularity=w.out, requantize=True, scale_fmt=UE)
    try:
        fp8_regimes.assert_requant_torch_cuda(y, ys, q, s, w.sg, w.dst, w.out, UE)
        assert_lossless(q, s, w.sg, y.view(torch.uint8).cpu().numpy(), ys.cpu().numpy(), w.out, *w.dst)
        assert all(guards_intact(b) for b in bases)
    finally:
        sync.close()
        cleanup(sources)


def source_values(sources, boxes, g, shape):
    """The values f32(q) * s of UE8M0 source-quantised shards, assembled over the global shape."""
    out = torch.full(shape, float("nan"), device=DEV)
    for (src, *_), (off, loc) in zip(sources, boxes):
        q, s, _ = src._quantized["w"]
        e = torch.from_numpy(np.ascontiguousarray(expand(s.cpu().numpy(), tuple(loc), g, off[-2], off[-1]))).to(DEV)
        out[tuple(slice(o, o + n) for o, n in zip(off, loc))] = q.float() * e
    return out


CONTAINED = {  # name -> (source granularity, source boxes of a [300, 512] tensor, destination window, granularity)
    "channel_from_block": ("block", (((0, 0), (128, 512)), ((128, 0), (172, 512))), ((0, 128), (300, 128)), "channel"),
    "block_from_one_tensor_shard": ("tensor", (((0, 0), (300, 512)),), ((37, 70), (200, 300)), "block"),
    "channel_from_one_tensor_shard": ("tensor", (((0, 0), (300, 512)),), ((0, 0), (300, 512)), "channel"),
    "tp_block_cut_at_128_columns": ("block", (((0, 0), (300, 256)), ((0, 256), (300, 256))), ((0, 256), (300, 256)), "block"),
}


@pytest.mark.parametrize("case", sorted(CONTAINED))
def test_lossless_requantise_of_contained_groups(case):
    sg, boxes, (off, loc), dg = CONTAINED[case]
    full = u8.synth_f32((300, 512), 40 + len(case), spread=12).to(torch.bfloat16)
    sources, handles = register_boxes(full, boxes, quantize={"w": sg}, scale_fmt=UE)
    try:
        before = source_values(sources, boxes, sg, (300, 512))[tuple(slice(o, o + n) for o, n in zip(off, loc))]
        sync, y, ys, bases = pull_box(handles, (300, 512), (off, loc), E4M3, granularity=dg, requantize=True,
                                      scale_fmt=UE)
        e = torch.from_numpy(np.ascontiguousarray(expand(ys.cpu().numpy(), tuple(loc), dg))).to(DEV)
        after = y.float() * e
        assert torch.isfinite(before).all() and torch.equal(after.view(torch.int32), before.view(torch.int32))
        s_src = torch.cat([src._quantized["w"][1].reshape(-1) for src, *_ in sources])
        assert ys.max() <= s_src.max()
        assert all(guards_intact(b) for b in bases)
        sync.close()
    finally:
        cleanup(sources)


@pytest.mark.parametrize("g", u8.GRANULARITIES)
def test_published_ue8m0_handles_requantised_into_their_own_layout_keep_their_values(g):
    full = u8.synth_f32((300, 512), 44, spread=12).to(torch.bfloat16)
    boxes = (((0, 0), (300, 256)), ((0, 256), (300, 256)))  # column shards cut on a block boundary
    sources, handles = register_boxes(full, boxes, quantize={"w": g}, scale_fmt=UE)
    try:
        want = source_values(sources, boxes, g, (300, 512))
        for off, loc in boxes:
            sync, y, ys, _ = pull_box(handles, (300, 512), (off, loc), E4M3, granularity=g, requantize=True,
                                      scale_fmt=UE)
            e = torch.from_numpy(np.ascontiguousarray(expand(ys.cpu().numpy(), tuple(loc), g))).to(DEV)
            assert torch.equal((y.float() * e).view(torch.int32), region(want, off, loc).view(torch.int32)), off
            sync.close()
    finally:
        cleanup(sources)


# ---- both ends of the domain -------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", (torch.bfloat16, torch.float32), ids=lambda d: str(d)[6:])
def test_amax_at_the_dtype_top_reads_back_as_inf(dtype):
    """amax >= 248 * 2^120: scale_inv 2^120 and q = 256, so f32(q) * scale_inv = 2^128 overflows to +Inf; a
    dequantising pull gives +Inf there and a requantising pull the NaN and zero pattern of the torch composition."""
    top = float(torch.finfo(dtype).max)
    assert top >= 248 * 2.0 ** 120
    x = (u8.synth_f32((128, 256), 3) * 0.01).to(dtype)
    x[5, 9] = top
    src = DirectWeightSyncSource()
    try:
        h = src.register({"w": x.to(DEV)}, rank=0, quantize={"w": "block"}, scale_fmt=UE)["w"]
        q, s, _ = src._quantized["w"]
        assert_exact(q, s, x, "block", 0, 0, UE)
        assert float(s[0, 0]) == 2.0 ** 120 and float(q[5, 9].float()) == 256.0
        y = torch.zeros(x.shape, dtype=dtype, device=DEV)
        sync = DirectWeightSyncDest()
        run(sync.pull({"w": [h]}, {"w": y}))
        sync.close()
        assert torch.equal(y, torch_dequantize(q, s, "block", 0, 0, dtype))
        assert y[5, 9] == float("inf") and torch.isfinite(y[:, 128:]).all()
        sync, yq, ys, bases = pull_box([h], tuple(x.shape), whole(tuple(x.shape)), E4M3, granularity="block",
                                       requantize=True, scale_fmt=UE)
        sync.close()
        want_q, want_s = u8.torch_requantize(q, s, "block", 0, 0, "block", scale_fmt=UE)
        assert torch.equal(yq.view(torch.uint8), want_q.view(torch.uint8))
        assert torch.equal(ys.view(torch.int32), want_s.view(torch.int32))
        b = yq.view(torch.uint8)[:, :128]
        assert torch.isinf(ys[0, 0]) and b[5, 9] & 0x7F == 0x7F and ((b & 0x7F) == 0x7F).sum() == 1
        assert ((b & 0x7F) == 0).sum() == b.numel() - 1  # every finite element +-0
    finally:
        run(src.cleanup())


def test_source_scale_under_2_pow_22_loses_low_bits_as_torch_does():
    """A block source scale of 2^-23 over small |q|: the destination's clamp picks s' = 2^-22 > s, and the odd
    subnormal bytes lose their low bit, exactly as the torch composition does."""
    q = torch.arange(0, 128, dtype=torch.uint8).repeat(128, 2)[:, :256] & 0x8F  # +-subnormal and small normal bytes
    s = torch.tensor([[2.0 ** -23, 2.0 ** -3]])
    sources, handles = register_boxes(q.view(E4M3), [whole((128, 256))], granularity="block",
                                      scale_of=partial(dq_local_scale, s, "block"))
    sync, y, ys, _ = pull_box(handles, (128, 256), whole((128, 256)), E4M3, granularity="block", requantize=True,
                              scale_fmt=UE)
    try:
        fp8_regimes.assert_requant_torch_cuda(y, ys, q.view(E4M3), s, "block", whole((128, 256)), "block", UE)
        assert float(ys[0, 0]) == 2.0 ** -22
        before = q.view(E4M3).float()[:, :128] * 2.0 ** -23
        after = y.cpu().float()[:, :128] * 2.0 ** -22
        assert not torch.equal(after, before)
        assert_lossless(q.view(E4M3), s, "block", y.view(torch.uint8).cpu().numpy()[:, 128:], ys.cpu().numpy()[:, 1:], "block",
                        (0, 128), (128, 128))
    finally:
        sync.close()
        cleanup(sources)


# ---- a state-dict round trip -------------------------------------------------------------------------
def test_put_and_get_state_dict_with_ue8m0_scales():
    import torch.distributed as dist
    from torch.testing._internal.distributed.fake_pg import FakeStore

    async def main():
        dist.init_process_group("fake", store=FakeStore(), rank=0, world_size=1)
        await ts.initialize()
        try:
            src = {"a": u8.synth_f32((256, 384), 91).to(torch.bfloat16).to(DEV),
                   "b": u8.synth_f32((2, 130, 260), 92).to(torch.bfloat16).to(DEV),
                   "norm": torch.randn(384, device=DEV).to(torch.bfloat16)}
            quant = {"a": "block", "b": "channel"}
            await ts.put_state_dict(src, "policy_ue8m0", direct_rdma=True, quantize=quant, scale_fmt=UE)
            deq = {"a": torch.zeros(256, 384, dtype=torch.bfloat16, device=DEV),
                   "b": torch.zeros(2, 130, 260, dtype=torch.bfloat16, device=DEV),
                   "norm": torch.zeros(384, dtype=torch.bfloat16, device=DEV)}
            rq = {"a": torch.zeros(256, 384, dtype=E4M3, device=DEV), "b": torch.zeros(2, 130, 260, dtype=E4M3, device=DEV),
                  "norm": torch.zeros(384, dtype=torch.bfloat16, device=DEV)}
            bs = {"a": torch.zeros(2, 3, device=DEV), "b": torch.zeros(2, 2, 3, device=DEV)}
            for _ in range(2):
                assert await ts.get_state_dict("policy_ue8m0", user_state_dict=deq, direct_rdma=True) is deq
                for n, g in quant.items():
                    q, s = u8.torch_quantize(src[n], g, scale_fmt=UE)
                    assert torch.equal(deq[n], torch_dequantize(q, s, g, 0, 0, torch.bfloat16)), n
                    assert ((s.view(torch.int32) & 0x7FFFFF) == 0).all()
                assert torch.equal(deq["norm"], src["norm"])
                await ts.get_state_dict("policy_ue8m0", user_state_dict=rq, direct_rdma=True, block_scales=bs, requantize=True,
                                        scale_fmt=UE)
                for n, g in quant.items():
                    q, s = u8.torch_quantize(src[n], g, scale_fmt=UE)
                    want_q, want_s = u8.torch_requantize(q, s, g, 0, 0, "block", scale_fmt=UE)
                    assert torch.equal(rq[n].view(torch.uint8), want_q.view(torch.uint8)), n
                    assert torch.equal(bs[n].view(torch.int32), want_s.reshape(bs[n].shape).view(torch.int32)), n
                src["a"].mul_(0.5)
                src["b"].mul_(3.0)
                await ts.put_state_dict(None, "policy_ue8m0", direct_rdma=True)
        finally:
            await ts.shutdown()
            dist.destroy_process_group()

    run(main())

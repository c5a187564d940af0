"""The packed-destination regimes (tests/packed_regimes.py) without a GPU: every regime on every route it takes,
planned on host memory, compiled with the host compilers and replayed with the oracle interpreters, equals the
numpy reference bit for bit (bytes and scales, sentinels outside every part); each regime reaches the branch it is
named for; the refusals of packed pulls are pinned; and a few hundred random specs replay to the reference."""

import asyncio

import numpy as np
import pytest
import torch

from tests import packed_regimes as pr
from tests.helpers import cuda_like
from torchstore_b200 import _native
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, PackedPart, _build_named
from torchstore_b200.launch import Plans
from torchstore_b200.planner import StridedMem, build_rects

# Every regime the catalogue names.  A regime added there, or dropped from it, fails test_catalogue_is_complete
# until this list says so too.
EXPECTED = ["col_parts", "drop_col_dim", "drop_row_dim", "drop_two_lead", "holes", "kv_replicated", "mixed_routes",
            "mixed_routes_ue8m0_verbatim", "per_tensor_sources", "row_parts_unaligned", "sharded_sources", "src_phase",
            "w13_straddle"]


def test_catalogue_is_complete():
    assert sorted(pr.REGIMES) == EXPECTED
    for name, r in pr.REGIMES.items():
        assert r.branch_route in r.routes, name
        assert all(ro in pr.ROUTES for ro in r.routes) or r.custom is not None, name
    kinds = {pr.ROUTES[ro].kind for _, ro in pr.CASES if ro in pr.ROUTES}
    assert kinds == {"copy", "cast", "quant", "dequant", "requant", "verbatim"}


def run_case(regime, route, variant, seed=11):
    spec = pr.spec(regime, route)
    data = pr.make_data(spec, seed, special=variant == "special")
    run = pr.host_pull(spec, data)
    pr.assert_pull(spec, run.result(), pr.expect(spec, data), f"{regime}/{route}/{variant}")
    if variant == "update":
        # the same tables, replayed after the sources changed in place, give the new values
        new = pr.make_data(spec, seed + 1000)
        pr.refill(spec, run.handles, new, lambda b: b.shard, lambda b: b.scale)
        run.replay()
        pr.assert_pull(spec, run.result(), pr.expect(spec, new), f"{regime}/{route}/update")
    return run


@pytest.mark.parametrize("variant", pr.VARIANTS)
@pytest.mark.parametrize("regime,route", pr.CASES, ids=[f"{r}-{ro}" for r, ro in pr.CASES])
def test_regime_replays_to_the_reference(regime, route, variant):
    run_case(regime, route, variant)


@pytest.mark.parametrize("regime", sorted(pr.REGIMES))
def test_regime_reaches_its_branch(regime):
    r = pr.REGIMES[regime]
    run = run_case(regime, r.branch_route, "finite")
    assert r.holds(run), f"{regime} ({r.doc}) not reached on {r.branch_route}"


def test_drop_col_dim_lifts_a_stride_zero_dim_on_the_quantising_routes():
    for route in ("quant_fp8_block_bfloat16", "quant_int8_channel_bfloat16", "quant_ue8m0_tensor_float16"):
        run = run_case("drop_col_dim", route, "finite")
        assert pr.REGIMES["drop_col_dim"].holds(run), route


def test_special_values_reach_every_part():
    """The special variant plants a value at some spot of every part (and at group edges inside them)."""
    for regime in ("row_parts_unaligned", "col_parts", "drop_two_lead", "sharded_sources"):
        spec = pr.spec(regime, "copy_bf16")
        assert {n for n, _ in pr.spots(spec)} == {p.source for p in spec.dests["w"].parts}, regime
        finite, special = pr.make_data(spec, 3), pr.make_data(spec, 3, special=True)
        for n in spec.sources:
            assert not torch.equal(finite.full[n], special.full[n]), (regime, n)
        assert not all(special.full[n].float().isfinite().all() for n in spec.sources), regime


# ---- refusals ---------------------------------------------------------------------------------------------------------
def host_setup(spec, data=None):
    data = data or pr.make_data(spec, 1)
    handles = pr.handles_of(spec, data, pr.HostBuffer)
    dests, scales, slices = pr.dests_of(spec)
    return data, handles, dests, scales, slices


@pytest.mark.parametrize("regime,dim", [("drop_row_dim", "row"), ("drop_col_dim", "column")])
@pytest.mark.parametrize("q", pr.SCALED)
def test_verbatim_with_a_dropped_row_or_column_dim_is_refused(regime, dim, q):
    r = pr.REGIMES[regime]
    srcs = {n: pr.Src(shape, q, "block", boxes) for n, (shape, boxes) in r.sources.items()}
    spec = pr.Spec(srcs, {"w": pr.Dst(r.shape, q, "block", r.parts)}, verbatim=True)
    _, handles, dests, scales, slices = host_setup(spec)
    scaled, _ = pr.verdicts(spec, handles, dests, scales)
    assert scaled["w"][-1] == "verbatim"
    ops = DirectWeightSyncDest()._build_plan(handles, dests, slices, packed=spec.packed())
    with pytest.raises(ValueError, match=r"verbatim pull of 'w' \(block_scales\): a packed part whose int index drops "
                                         r"one of the destination's last two dims cannot keep its source's scale groups"):
        DirectWeightSyncDest._verbatim_rects(ops, scaled)


@pytest.mark.parametrize("route", ["dq_e4m3_block_bfloat16", "dq_int8_channel_float32", "rq_block_channel",
                                   "rq_tensor_block"])
def test_scaled_sources_into_a_dropped_column_dim_are_refused(route):
    """dest[R, C, 2] at [..., k] from scaled handles: the dequantising and requantising kernels move whole source rows
    into whole destination rows, and such a part gives each destination row one element of a source row.  pull()
    refuses it with a ValueError naming the destination and the part before anything is compiled."""
    r, ro = pr.REGIMES["drop_col_dim"], pr.ROUTES[route]
    spec = pr.Spec({n: pr.Src(shape, ro.src, ro.sg, boxes) for n, (shape, boxes) in r.sources.items()},
                   {"w": pr.Dst(r.shape, ro.out, ro.g, r.parts)}, requantize=ro.kind == "requant")
    match = pr.refusal(spec)
    assert match and "part 0 \\(source 's0'\\)" in match
    _, handles, dests, scales, _ = host_setup(spec)
    if ro.kind == "requant":  # the scaled destination's checks read only metadata: claim CUDA
        dests = {n: cuda_like(t) for n, t in dests.items()}
    sync = DirectWeightSyncDest()
    with pytest.raises(ValueError, match=match):
        asyncio.run(sync.pull(handles, dests, packed=spec.packed(), requantize=spec.requantize,
                              **{k: v or None for k, v in scales.items()}))
    assert sync._plan is None
    # the same part on a quantising route is taken
    run_case("drop_col_dim", "quant_fp8_channel_float16", "finite")


def holed_spec(route):
    r, ro = pr.REGIMES["holes"], pr.ROUTES[route]
    return pr.Spec({n: pr.Src(shape, ro.src, ro.sg, boxes) for n, (shape, boxes) in r.sources.items()},
                   {"w": pr.Dst(r.shape, ro.out, ro.g, r.parts)}, requantize=ro.kind == "requant")


@pytest.mark.parametrize("route", ["quant_fp8_block_bfloat16", "quant_fp8_channel_float16", "quant_int8_tensor_float32",
                                   "rq_block_block"])
def test_grouped_route_with_a_hole_is_refused_naming_the_weight(route):
    """The host compiler refuses the uncovered destination group naming its target, which the pull's plan builder
    turns into a ValueError naming the weight."""
    spec = holed_spec(route)
    with pytest.raises(_native.TsbError, match="target 0"):
        pr.host_pull(spec, pr.make_data(spec, 4))
    calls = []

    def build(per_device):
        calls.append(per_device)
        return pr.host_pull(spec, pr.make_data(spec, 4))

    with pytest.raises(ValueError, match=r"^pull of 'w': .*target 0"):
        _build_named(Plans(), build, {0: None}, {"target": ["w"]}, lambda n: f"pull of '{n}'")
    assert calls == [{0: None}]


def mixed_handles(first, second, dest_dtype, dest_g=None, requantize=False):
    """A packed name whose part 0 reads ``first`` (dtype, granularity) handles and part 1 ``second``: the route
    checks take the union, so a mix is refused even though part 0 alone would pass."""
    srcs = {"a": pr.Src((64, 128), first[0], first[1], pr.shard((64, 128), 0, 2)),
            "b": pr.Src((64, 128), second[0], second[1], pr.whole((64, 128)))}
    parts = (PackedPart("a", (slice(0, 64), slice(0, 128)), (0, 0)), PackedPart("b", (slice(64, 128), slice(0, 128)), (0, 0)))
    spec = pr.Spec(srcs, {"w": pr.Dst((128, 128), dest_dtype, dest_g, parts)}, requantize=requantize)
    return spec, host_setup(spec)


@pytest.mark.parametrize("first,second,match", [
    (("e4m3", "block"), ("e4m3", "channel"), r"the handles of 'w' mix scale granularities \['block', 'channel'\]"),
    (("e4m3", "tensor"), ("bfloat16", None), "the handles of 'w' mix scaled fp8 and unscaled sources"),
    (("int8", "channel"), ("e4m3", "channel"), "the handles of 'w' mix scaled int8 and scaled fp8 sources"),
])
def test_dequantising_parts_mixing_handle_kinds_are_refused(first, second, match):
    spec, (_, handles, dests, _, _) = mixed_handles(first, second, "bfloat16")
    with pytest.raises(ValueError, match=match):
        asyncio.run(DirectWeightSyncDest().pull(handles, dests, packed=spec.packed()))


@pytest.mark.parametrize("first,second,exc,match", [
    (("e4m3", "block"), ("e4m3", "tensor"), ValueError,
     r"the handles of block-scaled destination 'w' mix scale granularities \['block', 'tensor'\] \(requantize=True\)"),
    (("e4m3", "block"), ("bfloat16", None), ValueError,
     r"the handles of block-scaled destination 'w' mix scaled fp8 and unscaled sources \(requantize=True\)"),
    (("int8", "block"), ("e4m3", "block"), ValueError,
     "the handles of block-scaled destination 'w' mix scaled int8 and scaled fp8 sources"),
    (("bfloat16", None), ("float32", None), TypeError, r"block-scaled pulls of 'w' read bf16, f16 or f32 handles of one dtype"),
])
def test_grouped_parts_mixing_handle_kinds_are_refused(first, second, exc, match):
    spec, (_, handles, dests, scales, _) = mixed_handles(first, second, "e4m3", "block", requantize=True)
    with pytest.raises(exc, match=match):
        pr.verdicts(spec, handles, dests, scales)


# ---- random specs --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("chunk", range(10))
def test_random_specs_replay_to_the_reference(chunk):
    for seed in range(30 * chunk, 30 * (chunk + 1)):
        spec = pr.random_spec(seed)
        data, handles, dests, _, _ = host_setup(spec, pr.make_data(spec, seed, special=seed % 3 == 0))
        assert DirectWeightSyncDest._check_packed(handles, dests, spec.packed())  # the generator makes valid specs
        if pr.refusal(spec):
            with pytest.raises(ValueError, match=pr.refusal(spec)):
                pr.host_pull(spec, data)
            continue
        run = pr.host_pull(spec, data)
        pr.assert_pull(spec, run.result(), pr.expect(spec, data), f"random spec {seed}")


def test_random_specs_draw_every_kind():
    specs = [pr.random_spec(s) for s in range(300)]
    ranks = {len(s.dests["w"].shape) for s in specs}
    dropped = [d for s in specs for p in s.dests["w"].parts for d, e in enumerate(p.dest_index) if isinstance(e, int)]
    assert ranks == {2, 3, 4}
    assert {d for d in dropped} >= {0, 1, 2}  # ints on leading, row and column dims
    layouts = [len(src.boxes) for s in specs for src in s.sources.values()]
    assert min(layouts) == 1 and max(layouts) >= 4
    assert any(len(set(src.boxes)) < len(src.boxes) for s in specs for src in s.sources.values())  # replicas
    assert {s.route_of("w") for s in specs} == {"copy", "cast", "quant", "dequant", "requant"}
    refused = [s for s in specs if pr.refusal(s)]
    assert 0 < len(refused) < len(specs) // 10  # dequantising and requantising parts dropping the last dim
    assert any(np.prod(s.dests["w"].shape) > sum(np.prod([1 if isinstance(e, int) else e.stop - e.start
                                                           for e in p.dest_index]) for p in s.dests["w"].parts)
               for s in specs)  # holes


def test_host_windows_of_a_dropped_dim_are_stride_zero():
    """op_windows lifts a dropped dim as a unit dim of stride 0 on the source side (it never addresses memory)."""
    spec = pr.spec("drop_two_lead", "copy_bf16")
    _, handles, dests, _, slices = host_setup(spec)
    for op in DirectWeightSyncDest()._build_plan(handles, dests, slices, packed=spec.packed()):
        src, dst = DirectWeightSyncDest.op_windows(op, StridedMem.from_tensor(op.rdma_buffer.shard))
        assert op.dest_dropped == (0, 1) and src.shape == dst.shape
        assert [src.stride[d] for d in op.dest_dropped] == [0, 0]
        rects, n = build_rects([(src, dst)])
        assert n == 1

"""Power-of-two (UE8M0) scales on the H100: quantising pulls, requantising pulls and source-side quantisation with
``scale_fmt="ue8m0"``, bit for bit against the torch-CUDA rendering of the formula (ue8m0_oracle, NaN bytes and
scale_inv included) and against the numpy oracle on finite groups; non-finite groups; plan rebuilds when the format
changes; and the lossless round trip of power-of-two groups requantised onto themselves.  Several "ranks" are
emulated as several sources on cuda:0."""

import numpy as np
import pytest
import torch

from oracle.dequant_fp8_oracle import expand
from oracle.ue8m0_oracle import GRANULARITIES, bits_of, quantize, synth_f32, torch_quantize, torch_requantize, widen
from tests.fp8_regimes import whole
from tests.helpers import DEV, E4M3, KW, cleanup, pull_box, run
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource, ScaledNvlinkBuffer
from torchstore_b200.transport.types import TensorSlice

pytestmark = pytest.mark.gpu
DTYPES = (torch.bfloat16, torch.float16, torch.float32)


def dest_scale(g: str, shape) -> torch.Tensor:
    *lead, n, k = shape
    return torch.full({"block": (*lead, -(-n // 128), -(-k // 128)), "channel": (*lead, n, 1), "tensor": tuple(lead)}[g],
                      -1.0, device=DEV)


def publish(full: torch.Tensor, boxes, **register_kw):
    """One source per box (offsets, extents) of `full`, registered on cuda:0 -> (sources, handles)."""
    sources, handles = [], []
    for r, (off, loc) in enumerate(boxes):
        shard = full[tuple(slice(o, o + e) for o, e in zip(off, loc))].contiguous().to(DEV)
        ts = TensorSlice(tuple(off), (r,), tuple(full.shape), tuple(loc), (len(boxes),))
        src = DirectWeightSyncSource()
        handles.append(src.register({"w": shard}, rank=r, tensor_slices={"w": ts}, **register_kw)["w"])
        sources.append((src, shard))
    return sources, handles


def rows(shape, k):
    """FSDP(k) row boxes of the last-but-one dim (the last box takes the remainder)."""
    n = shape[-2]
    cuts = [i * n // k for i in range(k)] + [n]
    lead = tuple(0 for _ in shape[:-2])
    return [(lead + (a, 0), tuple(shape[:-2]) + (b - a, shape[-1])) for a, b in zip(cuts, cuts[1:])]


def cols(shape, cuts):
    """Column boxes of the last dim at `cuts`."""
    lead = tuple(0 for _ in shape[:-2])
    edges = [0] + list(cuts) + [shape[-1]]
    return [(lead + (0, a), tuple(shape[:-1]) + (b - a,)) for a, b in zip(edges, edges[1:])]


def assert_exact(q, s, x, g, r0=0, c0=0):
    """Bit-exact with torch CUDA (NaN bytes and scale_inv included), and with the numpy oracle on finite groups."""
    tq, ts = torch_quantize(x.to(DEV), g, r0, c0, scale_fmt="ue8m0")
    assert torch.equal(q.view(torch.uint8), tq.view(torch.uint8))
    assert torch.equal(s.view(torch.int32), ts.reshape(s.shape).view(torch.int32))
    want_q, want_s = quantize(widen(bits_of(x.cpu()), str(x.dtype)[6:]), g, r0, c0, scale_fmt="ue8m0")
    got_q, got_s = q.view(torch.uint8).cpu().numpy(), s.cpu().numpy().reshape(want_s.shape)
    fin = np.isfinite(expand(want_s, want_q.shape, g, r0, c0))
    assert np.array_equal(got_q[fin], want_q[fin])
    fs = np.isfinite(want_s)
    assert np.array_equal(got_s[fs].view(np.uint32), want_s[fs].view(np.uint32))
    assert (got_s[fs].view(np.uint32) & 0x7FFFFF == 0).all()  # powers of two


# ---- quantising pulls ------------------------------------------------------------------------------------------
LAYOUTS = {
    "exact_300x520": ((300, 520), lambda s: [((0, 0), s)]),
    "fsdp2_rows": ((512, 384), lambda s: rows(s, 2)),
    "fsdp4_rows_ragged_300x200": ((300, 200), lambda s: rows(s, 4)),
    "fsdp4_cols": ((256, 512), lambda s: cols(s, (128, 256, 384))),
    "unaligned_cols_at_70_and_201": ((260, 330), lambda s: cols(s, (70, 201))),  # scalar paths: sources not 16-byte aligned
    "moe_3x130x260": ((3, 130, 260), lambda s: [((0, 0, 0), s)]),
    "moe_rows_3x130x260": ((3, 130, 260), lambda s: rows(s, 2)),
}


@pytest.mark.parametrize("layout", sorted(LAYOUTS))
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("g", GRANULARITIES)
def test_quantising_pull_is_exact(g, dtype, layout):
    shape, boxes = LAYOUTS[layout]
    full = synth_f32(shape, 101 + len(layout)).to(dtype)
    sources, handles = publish(full, boxes(shape))
    sync, q, s, _ = pull_box(handles, shape, whole(shape), E4M3, granularity=g, scale_fmt="ue8m0")
    sync.close()
    assert_exact(q, s, full, g)
    cleanup(sources)


@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
def test_long_channel_rows_take_the_two_pass_path(dtype):
    shape = (3, 16400 if dtype != torch.float32 else 8200)  # over the 32 KiB row stage
    full = synth_f32(shape, 7).to(dtype)
    sources, handles = publish(full, cols(shape, (shape[1] // 2,)))
    sync, q, s, _ = pull_box(handles, shape, whole(shape), E4M3, granularity="channel",
                             scale_fmt="ue8m0")
    sync.close()
    assert_exact(q, s, full, "channel")
    cleanup(sources)


@pytest.mark.parametrize("g", GRANULARITIES)
def test_non_finite_groups(g):
    """An Inf group: scale_inv Inf, its finite elements +-0 and its Infs NaN.  A NaN group: NaN scale and bytes."""
    full = synth_f32((260, 300), 8).to(torch.bfloat16)
    full[3, 5] = float("inf")
    full[200, 140] = float("nan")
    sources, handles = publish(full, rows(full.shape, 2))
    sync, q, s, _ = pull_box(handles, tuple(full.shape), whole(tuple(full.shape)), E4M3, granularity=g,
                             scale_fmt="ue8m0")
    sync.close()
    assert_exact(q, s, full, g)
    sc = s.cpu()
    assert torch.isnan(sc).any()
    if g != "tensor":
        inf_group = sc[0, 0] if g == "block" else sc[3, 0]
        assert torch.isinf(inf_group)
        qb = q.view(torch.uint8).cpu()
        assert qb[3, 5] & 0x7F == 0x7F and qb[3, 6] & 0x7F == 0  # the Inf is NaN, a finite neighbour +-0
    cleanup(sources)


def test_switching_the_format_rebuilds_the_plan():
    """None, then "ue8m0", then None on the same destination: each result is its own formula and every change
    compiles new plans."""
    full = synth_f32((300, 260), 9).to(torch.bfloat16)
    sources, handles = publish(full, rows(full.shape, 2))
    qs = {g: torch.zeros(full.shape, dtype=E4M3, device=DEV) for g in GRANULARITIES}
    ss = {g: dest_scale(g, full.shape) for g in GRANULARITIES}
    d = DirectWeightSyncDest()
    seen = set()
    for fmt in (None, "ue8m0", None):
        run(d.pull({f"w_{g}": handles for g in GRANULARITIES}, {f"w_{g}": qs[g] for g in GRANULARITIES},
                   **{KW[g]: {f"w_{g}": ss[g]} for g in GRANULARITIES}, scale_fmt=fmt))
        ids = set(d._block_plans.values()) | set(d._scaled_plans.values())
        assert ids and not ids & seen
        seen |= ids
        for g in GRANULARITIES:
            tq, ts = torch_quantize(full.to(DEV), g, scale_fmt=fmt)
            assert torch.equal(qs[g].view(torch.uint8), tq.view(torch.uint8)), (fmt, g)
            assert torch.equal(ss[g].view(torch.int32), ts.reshape(ss[g].shape).view(torch.int32)), (fmt, g)
        # the same format again replays the cached plans
        run(d.pull({f"w_{g}": handles for g in GRANULARITIES}, {f"w_{g}": qs[g] for g in GRANULARITIES},
                   **{KW[g]: {f"w_{g}": ss[g]} for g in GRANULARITIES}, scale_fmt=fmt))
        assert set(d._block_plans.values()) | set(d._scaled_plans.values()) == ids
    d.close()
    cleanup(sources)


# ---- requantising pulls -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("dg", GRANULARITIES)
@pytest.mark.parametrize("sg", GRANULARITIES)
def test_requantising_pull_is_the_torch_composition(sg, dg):
    """Float32-scaled fp8 handles (FSDP(2) row shards, the cut mid-block) requantised into UE8M0 destinations:
    bit-exact with dequantising to f32, then the UE8M0 quantise."""
    x = synth_f32((300, 260), 10 + len(sg + dg)).to(torch.bfloat16).to(DEV)
    q_full, s_full = torch_quantize(x, sg)
    boxes = rows(x.shape, 2)
    sources, handles = [], []
    for r, (off, loc) in enumerate(boxes):
        r0, n = off[0], loc[0]
        shard = q_full[r0:r0 + n].contiguous()
        if sg == "block":
            scale = s_full[r0 // 128: -(-(r0 + n) // 128)].contiguous()
        else:
            scale = s_full[r0:r0 + n].contiguous() if sg == "channel" else s_full
        ts = TensorSlice(off, (r,), tuple(x.shape), loc, (2,))
        src = DirectWeightSyncSource()
        handles.append(src.register({"w": shard}, rank=r, tensor_slices={"w": ts}, **{KW[sg]: {"w": scale}})["w"])
        sources.append((src, shard))
    sync, q, s, _ = pull_box(handles, tuple(x.shape), whole(tuple(x.shape)), E4M3, granularity=dg, requantize=True,
                             scale_fmt="ue8m0")
    sync.close()
    tq, ts_ = torch_requantize(q_full, s_full, sg, 0, 0, dg, scale_fmt="ue8m0")
    assert torch.equal(q.view(torch.uint8), tq.view(torch.uint8))
    assert torch.equal(s.view(torch.int32), ts_.reshape(s.shape).view(torch.int32))
    assert ((s.view(torch.int32) & 0x7FFFFF) == 0).all()
    cleanup(sources)


# ---- source-side quantisation -----------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES, ids=lambda d: str(d)[6:])
@pytest.mark.parametrize("g", GRANULARITIES)
def test_source_side_fsdp8_mid_block_shards(g, dtype):
    """FSDP(8) row shards of 300 rows cut blocks mid-block: the staging is exact with shard-local groups anchored at
    the global origin, the handles stay float32-scaled ScaledNvlinkBuffers, and a dequantising pull into f32 of all
    eight reads q * s."""
    full = synth_f32((300, 264), 12).to(dtype)
    full[150, 9] = float("nan")
    boxes = rows(full.shape, 8)
    sources, handles = publish(full, boxes, quantize={"w": g}, scale_fmt="ue8m0")
    want = []
    for (src, shard), (off, _), h in zip(sources, boxes, handles):
        q, s, _ = src._quantized["w"]
        assert isinstance(h.rdma_buffer, ScaledNvlinkBuffer) and h.rdma_buffer.granularity == g and s.dtype == torch.float32
        assert_exact(q, s, shard, g, off[0], 0)
        want.append(q.float() * torch.from_numpy(np.ascontiguousarray(
            expand(s.cpu().numpy(), tuple(q.shape), g, off[0], 0))).to(DEV))
    y = torch.zeros(full.shape, device=DEV)
    d = DirectWeightSyncDest()
    run(d.pull({"w": handles}, {"w": y}))
    d.close()
    want = torch.cat(want)
    assert torch.equal(torch.isnan(y), torch.isnan(want)) and torch.isnan(want).any()
    assert torch.equal(y.nan_to_num(0.0).view(torch.int32), want.nan_to_num(0.0).view(torch.int32))
    # refresh() keeps the format
    for src, shard in sources:
        shard.mul_(3)
        src.refresh()
    for (src, shard), (off, _) in zip(sources, boxes):
        q, s, _ = src._quantized["w"]
        assert_exact(q, s, shard, g, off[0], 0)
    cleanup(sources)


# ---- the lossless round trip ------------------------------------------------------------------------------------
@pytest.mark.parametrize("g", ("block", "channel"))
def test_power_of_two_groups_requantised_onto_themselves_keep_every_value(g):
    """UE8M0 source handles whose shard boundaries sit on group boundaries, requantised with UE8M0 into destinations
    whose groups coincide with the source groups: f32(q') * s' == f32(q) * s element for element."""
    full = synth_f32((512, 640), 13, spread=12).to(torch.bfloat16)
    boxes = rows(full.shape, 4)  # 128-row shards: block rows and channel rows coincide on both sides
    sources, handles = publish(full, boxes, quantize={"w": g}, scale_fmt="ue8m0")
    sync, q, s, _ = pull_box(handles, tuple(full.shape), whole(tuple(full.shape)), E4M3, granularity=g,
                             requantize=True, scale_fmt="ue8m0")
    sync.close()
    src_q = torch.cat([src._quantized["w"][0].view(torch.uint8) for src, _ in sources]).view(E4M3)
    src_s = torch.cat([src._quantized["w"][1] for src, _ in sources])
    before = src_q.float() * torch.from_numpy(np.ascontiguousarray(expand(src_s.cpu().numpy(), tuple(full.shape), g))).to(DEV)
    after = q.float() * torch.from_numpy(np.ascontiguousarray(expand(s.cpu().numpy(), tuple(full.shape), g))).to(DEV)
    assert torch.isfinite(before).all()
    assert torch.equal(after, before)
    assert (s <= src_s).all()
    cleanup(sources)

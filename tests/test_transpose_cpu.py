"""Transposed packed parts without a GPU: the validation of ``transpose`` and its route refusals before anything is
compiled, the field in the plan key and on the public path, the transpose oracle against torch, the planned ops of
FSDP(1) / FSDP(3) / uneven shards cut along each source dim replayed on host memory, the full-size Qwen3-30B-A3B
grouped experts at TP8 (every rank) and EP8, and the tile tables of tsb_transpose_compile_host replayed in numpy."""

import asyncio

import numpy as np
import pytest
import torch

import workloads
from oracle import packed_oracle, transpose_oracle as to
from tests.helpers import HostBuffer, fsdp_handles, handles_of
from tests.test_packed_cpu import ScaledHost
from torchstore_b200 import _native, state_dict_utils
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, PackedPart, RDMAWeightHandle, _packed_key
from torchstore_b200.planner import StridedMem, build_rects, build_transpose_rects
from torchstore_b200.transport.types import TensorSlice

QWEN = workloads.QWEN3_MOE
WHAT = r"packed destination 'fused' part 0 \(source 'a'\)"


def check(dest_shape, packed, handles, match):
    dests = {"fused": torch.zeros(dest_shape, dtype=torch.bfloat16)}
    with pytest.raises(ValueError, match=match):
        DirectWeightSyncDest._check_packed(handles, dests, packed)
    with pytest.raises(ValueError, match=match):
        asyncio.run(DirectWeightSyncDest().pull(handles, dests, packed=packed))


def T(index, offsets, **kw):
    return {"fused": (PackedPart("a", index, offsets, transpose=True, **kw),)}


# -- the oracle ----------------------------------------------------------------------------------------------------
def test_oracle_hand_written():
    """A 2x3 box at source offsets (1, 2) of a 4x5 source: box (i, j) reads source (1 + j, 2 + i)."""
    src = np.arange(20).reshape(4, 5)
    part = PackedPart("s", (slice(1, 4), slice(0, 2)), (1, 2), transpose=True)
    out = to.fill(np.full((5, 2), -1), [part], {"s": src})
    assert np.array_equal(out[1:4], [[7, 12], [8, 13], [9, 14]])
    assert (out[0] == -1).all() and (out[4] == -1).all()
    assert np.array_equal(to.read(src, (1, 2), (3, 2)), out[1:4])


@pytest.mark.parametrize("seed", range(4))
def test_oracle_matches_torch_transpose(seed):
    g = torch.Generator().manual_seed(seed)
    lead = [(), (3,), (2, 3)][seed % 3]
    a, b = (int(x) for x in torch.randint(1, 9, (2,), generator=g))
    src = torch.randn(lead + (b + 3, a + 2), generator=g)
    offs = (0,) * len(lead) + (3, 2)
    want = src[..., 3:, 2:].transpose(-2, -1).numpy()
    part = PackedPart("s", tuple(slice(0, e) for e in lead + (a, b)), offs, transpose=True)
    got = to.fill(np.zeros(lead + (a, b), dtype=np.float32), [part], {"s": src.numpy()})
    assert np.array_equal(got, want)
    assert np.array_equal(to.read(src.numpy(), offs, lead + (a, b)), want)
    parts, sources = to.plain([part], {"s": src.numpy()})
    assert np.array_equal(packed_oracle.fill(np.zeros(lead + (a, b), dtype=np.float32), parts, sources), want)


# -- validation ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("flag", [1, 0, "yes", None])
def test_transpose_must_be_a_bool(flag):
    check((4, 8), {"fused": (PackedPart("a", (slice(0, 4), slice(0, 8)), (0, 0), transpose=flag),)},
          {"a": handles_of((8, 4))}, WHAT + r": transpose must be a bool")


def test_source_needs_two_dims():
    check((4, 8), T((0, slice(0, 8)), (0,)), {"a": handles_of((8,))},
          WHAT + r": transpose swaps the source's last two dims, and the source has 1 dim")


def test_not_with_rotary():
    check((4, 8), T((slice(0, 4), slice(0, 8)), (0, 0), rotary_head_dim=4), {"a": handles_of((8, 4))},
          WHAT + r": transpose and rotary_head_dim do not combine")


@pytest.mark.parametrize("index", [(slice(0, 2), 1, slice(0, 4)), (slice(0, 2), slice(0, 4), 3)])
def test_int_index_must_not_drop_the_swapped_dims(index):
    check((2, 4, 4), T(index, (0, 0)), {"a": handles_of((2, 4))},
          WHAT + r": its int index drops one of the destination's last two dims")


def test_swapped_box_outside_the_source():
    # box (4, 6) reads a (6, 4) source box: at (0, 0) of an (8, 4) source it fits, at (3, 0) it leaves it
    check((4, 6), T((slice(0, 4), slice(0, 6)), (3, 0)), {"a": handles_of((8, 4))},
          WHAT + r": the source box at \(3, 0\) with extent \(6, 4\) leaves the source's global shape \(8, 4\)")
    DirectWeightSyncDest._check_packed({"a": handles_of((8, 4))}, {"fused": torch.zeros(4, 6)},
                                       T((slice(0, 4), slice(0, 6)), (2, 0)))


def test_hole_names_the_source_element():
    hs = {"a": handles_of((8, 4), n=2)[:1]}  # rows 0..4 only
    check((4, 6), T((slice(0, 4), slice(0, 6)), (0, 0)), hs, WHAT + r": no handle covers global element \(4, 0\)")


def test_routes_refuse_scaled_destinations_and_scaled_handles():
    hs = {"a": handles_of((8, 4))}
    dests = {"fused": torch.zeros(4, 8, dtype=torch.bfloat16)}
    parts = DirectWeightSyncDest._check_packed(hs, dests, T((slice(0, 4), slice(0, 8)), (0, 0)))
    for kw in ("block_scales", "channel_scales", "tensor_scales"):
        with pytest.raises(ValueError, match=WHAT + rf": a transposed part takes element-wise routes only .* is in {kw}"):
            DirectWeightSyncDest._check_transposed_routes(parts, {"fused": (kw, None, None, "quantise")})
    # dequantising: fp8 channel-scaled handles into a bf16 destination, refused in pull() before compiling
    shard = torch.zeros(8, 4, dtype=torch.uint8).view(torch.float8_e4m3fn)
    scaled = {"a": [RDMAWeightHandle(ScaledHost(shard, torch.ones(8, 1), "channel", 0, 0),
                                     TensorSlice((0, 0), (0,), (8, 4), (8, 4), (1,)), 0)]}
    with pytest.raises(ValueError, match=WHAT + r": a transposed part .* its source handles are scaled"):
        asyncio.run(DirectWeightSyncDest().pull(scaled, dests, packed=T((slice(0, 4), slice(0, 8)), (0, 0))))
    DirectWeightSyncDest._check_transposed_routes(parts, {})


def test_plan_key_tells_transpose_apart():
    def key(flag):
        return _packed_key({"w": (PackedPart("a", (slice(0, 4), slice(0, 4)), (0, 0), transpose=flag),)})
    assert key(True) != key(False) and key(True) == key(True)


def test_field_rides_in_packed_on_get_state_dict():
    hs = handles_of((8, 4), n=2)

    class Store:
        async def get(self, key):
            return 2

        async def get_batch(self, keys):
            return {k: {"a": h} for k, h in zip(keys, hs)}

    store = Store()
    dst = {"w": torch.zeros(4, 8, dtype=torch.bfloat16)}
    try:
        bad = {"w": (PackedPart("a", (slice(0, 4), slice(0, 8)), (0, 0), transpose=1),)}
        with pytest.raises(ValueError, match=r"packed destination 'w' part 0 \(source 'a'\): transpose must be a bool"):
            asyncio.run(state_dict_utils.get_state_dict(store, "k", dst, direct_rdma=True, packed=bad))
        good = {"w": (PackedPart("a", (slice(0, 4), slice(0, 8)), (0, 0), transpose=True),)}
        with pytest.raises(RuntimeError, match="direct weight sync writes GPU memory"):
            asyncio.run(state_dict_utils.get_state_dict(store, "k", dst, direct_rdma=True, packed=good))
    finally:
        state_dict_utils.reset_direct_cache(store)


# -- planner -------------------------------------------------------------------------------------------------------
def apply_ops(ops, dests):
    """Move every op as its windows say (host tensors, torch strided views)."""
    for op in ops:
        src, dst = DirectWeightSyncDest.op_windows(op, StridedMem.from_tensor(op.rdma_buffer.shard))
        s, d = (torch.as_strided(t, w.shape, w.stride, (w.ptr - t.untyped_storage().data_ptr()) // t.element_size())
                for t, w in ((op.rdma_buffer.shard, src), (dests[op.name], dst)))
        d.copy_(s)


@pytest.mark.parametrize("n,dim", [(1, 0), (3, 0), (3, 1), (3, 2), (5, 1)])
def test_ops_fill_what_the_oracle_says(n, dim):
    """A [7, 11, 13] source cut into n uneven shards along ``dim``; a [3, 2, 10, 9] destination whose parts are a
    transposed box (int index on dim 1), an untransposed one and a transposed one at odd offsets."""
    g = torch.Generator().manual_seed(n * 10 + dim)
    full = torch.randint(-2 ** 15, 2 ** 15, (7, 11, 13), generator=g, dtype=torch.int16)
    hs = {"a": handles_of((7, 11, 13), n, torch.int16, dim, full)}
    parts = (PackedPart("a", (slice(0, 3), 0, slice(0, 10), slice(0, 9)), (1, 1, 2), transpose=True),
             PackedPart("a", (slice(0, 3), 1, slice(0, 10), slice(0, 9)), (4, 1, 2)),
             PackedPart("a", (slice(0, 3), 1, slice(0, 10), slice(0, 1)), (2, 10, 3), transpose=True))
    dests = {"fused": torch.full((3, 2, 10, 9), -7, dtype=torch.int16)}
    # the third part overlaps the second: it fills a destination of its own
    dests2 = {"fused": torch.full((3, 2, 10, 9), -7, dtype=torch.int16)}
    for spec, d in (((parts[0], parts[1]), dests), ((parts[2],), dests2)):
        ops = DirectWeightSyncDest()._build_plan(hs, d, packed={"fused": spec})
        apply_ops(ops, d)
        want = to.fill(np.full((3, 2, 10, 9), -7, dtype=np.int16), spec, {"a": full.numpy()})
        assert np.array_equal(d["fused"].numpy(), want)
        # replicated regions are read once, each (part, handle) intersection is one op
        assert len(ops) == sum(1 for p in spec for h in hs["a"] if _meets(p, h, (3, 2, 10, 9)))


def _meets(part, h, shape):
    box = [e for e, s in zip(torch.empty(shape, device="meta")[part.dest_index].shape, shape)]
    ext = box[:-2] + box[:-3:-1] if part.transpose else box
    return all(max(o, a) < min(o + e, a + x) for o, e, a, x in
               zip(part.source_offsets, ext, h.tensor_slice.offsets, h.tensor_slice.local_shape))


def _qwen_ops(tp, rank, ep, n):
    layout = workloads.qwen3_moe_layout(QWEN, n_layers=1, with_embeddings=False, grouped_experts=True)
    vl = workloads.vllm_tp_layout(layout, QWEN, tp, rank, ep=ep)
    names = [k for k in vl if k.endswith(("w13_weight", "w2_weight"))]
    hs = fsdp_handles(layout, n, lambda name, off, loc: HostBuffer(None, loc, torch.bfloat16),
                      names=[k for k in layout if ".experts.w" in k])
    dests = {k: torch.empty(vl[k][0], dtype=torch.bfloat16, device="meta") for k in names}
    packed = {k: vl[k][1] for k in names}
    return vl, dests, packed, DirectWeightSyncDest()._build_plan(hs, dests, packed=packed)


@pytest.mark.parametrize("tp,rank,ep", [(8, r, False) for r in range(8)] + [(8, 0, True), (8, 5, True)])
def test_qwen3_30b_a3b_grouped_experts_full_size(tp, rank, ep):
    """Full-size Qwen3-30B-A3B grouped experts (128 x [2048, 768]), FSDP(8) -> vLLM TP8 (every rank) or EP8: the ops of
    each destination tile it exactly, and every op's corners read what the element rule says."""
    vl, dests, packed, ops = _qwen_ops(tp, rank, ep, 8)
    e_r, f_r = (16, 768) if ep else (128, 96)
    name = "model.layers.0.mlp.experts."
    assert vl[name + "w13_weight"][0] == (e_r, 2 * f_r, 2048) and vl[name + "w2_weight"][0] == (e_r, 2048, f_r)
    for dname, parts in packed.items():
        mine = [op for op in ops if op.name == dname]
        assert all(op.transpose for op in mine)
        total = 0
        for op in mine:
            ext = [s.stop - s.start for s in op.dest_slices]
            total += int(np.prod(ext))
            sstart = [s.start for s in op.src_slices]
            # the element rule at the op's first and last element: dest (..., i, j) <- src (..., j, i)
            part = next(p for p in parts if all(b.start <= d.start and d.stop <= b.stop
                                                for b, d in zip(p.dest_index, op.dest_slices)))
            box0 = [b.start for b in part.dest_index]
            for corner in (0, 1):
                d = [s.start if not corner else s.stop - 1 for s in op.dest_slices]
                rel = [a - b for a, b in zip(d, box0)]
                want = [o + r for o, r in zip(part.source_offsets, rel[:-2] + [rel[-1], rel[-2]])]
                got = [o + s + (0 if not corner else e - 1) for o, s, e in
                       zip(op.src_offsets, sstart, ext[:-2] + [ext[-1], ext[-2]])]
                assert got == want, (dname, corner)
        assert total == int(np.prod(vl[dname][0])), dname  # the ops of distinct handles are disjoint


# -- tsb_transpose_compile_host ------------------------------------------------------------------------------------
DTYPES = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}


def _replay(tiles, sbase, dbase, sb, db, n_dst, src_bytes, dst_bytes, allowed: set):
    """Move every tile's elements byte for byte (same element size); count writes per destination element; check
    every read and the 16-byte marks."""
    writes = np.zeros(n_dst, dtype=np.int64)
    for t in tiles:
        i = np.arange(t["rows"])[:, None]
        j = np.arange(t["cols"])[None, :]
        so = (int(t["src"]) - sbase) + i * sb + j * int(t["src_stride"])
        do = (int(t["dst"]) - dbase) + i * int(t["dst_stride"]) + j * db
        assert set(so.reshape(-1).tolist()) <= allowed, "a read outside the source rect"
        np.add.at(writes, (do // db).reshape(-1), 1)
        if sb == db:
            for k in range(sb):
                dst_bytes[do + k] = src_bytes[so + k]
        for side, base, stride, n, bit in (("src", sbase, "src_stride", t["cols"], 1), ("dst", dbase, "dst_stride", t["rows"], 2)):
            aligned = int(t[side]) % 16 == 0 and (n == 1 or int(t[stride]) % 16 == 0)
            assert not (t["vec"] & bit) or aligned, "a 16-byte access marked on an unaligned side"
            assert bool(t["vec"] & bit) == aligned
    return writes


@pytest.mark.parametrize("es", [1, 2, 4, 8])
@pytest.mark.parametrize("lead,a,b,off", [((), 37, 53, (3, 5)), ((), 64, 128, (0, 0)), ((3,), 1, 53, (0, 1, 2)),
                                          ((2,), 37, 1, (1, 4, 0)), ((2, 3), 65, 33, (1, 0, 7, 9)),
                                          ((1, 2), 5, 130, (0, 1, 2, 3))])
def test_compile_host_tables_replay_to_the_oracle(es, lead, a, b, off):
    """Odd extents and offsets, extent-1 dims, every element size, 3-D and 4-D batches: every destination element is
    written once, every read lies inside the source rect, 16-byte accesses are marked exactly where their side is
    aligned, and the replayed bytes equal the oracle."""
    dt = DTYPES[es]
    g = torch.Generator().manual_seed(es * 100 + a)
    sshape = tuple(o + e + 2 for o, e in zip(off, lead + (b, a)))
    src = torch.randint(0, 120, sshape, generator=g, dtype=torch.int64).to(dt)
    dst = torch.full(lead + (a, b), 121, dtype=dt)
    part = PackedPart("s", tuple(slice(0, e) for e in lead + (a, b)), off, transpose=True)
    sw = StridedMem.from_tensor(src)
    sbox = sw.sub(tuple(slice(o, o + e) for o, e in zip(off, lead + (b, a))))
    swin = StridedMem(sbox.ptr, lead + (a, b), sbox.stride[:-2] + sbox.stride[:-3:-1], dt, -1)
    rects, n = build_transpose_rects([(swin, StridedMem.from_tensor(dst))])
    tiles = _native.transpose_compile_host(0, rects, n)
    assert len(tiles) == int(np.prod(lead or (1,))) * -(-a // (64 if es <= 2 else 32)) * -(-b // (64 if es <= 2 else 32))
    sbytes = src.numpy().view(np.uint8).reshape(-1)
    dbytes = dst.numpy().view(np.uint8).reshape(-1)
    idx = np.indices(lead + (b, a)).reshape(len(sshape), -1)
    allowed = set((np.ravel_multi_index(tuple(i + o for i, o in zip(idx, off)), sshape) * es).tolist())
    writes = _replay(tiles, src.data_ptr(), dst.data_ptr(), es, es, dst.numel(), sbytes, dbytes, allowed)
    assert (writes == 1).all()
    want = to.fill(np.full(lead + (a, b), 121, dtype=dst.numpy().dtype), [part], {"s": src.numpy()})
    assert np.array_equal(dst.numpy(), want)


@pytest.mark.parametrize("sdt,ddt", [(torch.float32, torch.bfloat16), (torch.bfloat16, torch.float32),
                                     (torch.float16, torch.float8_e4m3fn), (torch.float8_e5m2, torch.float16),
                                     (torch.float64, torch.float32)])
def test_compile_host_cast_tables_cover_once(sdt, ddt):
    src = torch.zeros(3, 41, 70, dtype=torch.uint8).view(sdt) if sdt.itemsize == 1 else torch.zeros(3, 41, 70, dtype=sdt)
    dst = torch.zeros(3, 70, 41, dtype=torch.uint8).view(ddt) if ddt.itemsize == 1 else torch.zeros(3, 70, 41, dtype=ddt)
    sw = StridedMem.from_tensor(src)
    swin = StridedMem(sw.ptr, (3, 70, 41), (sw.stride[0], sw.stride[2], sw.stride[1]), sdt, -1)
    rects, n = build_transpose_rects([(swin, StridedMem.from_tensor(dst))])
    tiles = _native.transpose_compile_host(0, rects, n)
    assert set(tiles["src_dtype"]) == {_native.cast_code(sdt)} and set(tiles["dst_dtype"]) == {_native.cast_code(ddt)}
    sb, db = sdt.itemsize, ddt.itemsize
    allowed = set(range(0, src.numel() * sb, sb))
    writes = _replay(tiles, src.data_ptr(), dst.data_ptr(), sb, db, dst.numel(), None, None, allowed)
    assert (writes == 1).all()


def test_non_transposed_rects_and_unsupported_casts_name_the_rect():
    src = torch.zeros(8, 16, dtype=torch.bfloat16)
    dst = torch.zeros(8, 16, dtype=torch.bfloat16)
    plain, _ = build_rects([(StridedMem.from_tensor(src), StridedMem.from_tensor(dst))])
    plain_2d = build_transpose_rects([(StridedMem(src.data_ptr(), (8, 16), (16, 1), torch.bfloat16, -1),
                                       StridedMem.from_tensor(dst))])[0]
    with pytest.raises(_native.TsbError, match=r"rect 0: not a transposed rect: its source is not contiguous") as e:
        _native.transpose_compile_host(0, plain_2d, 1)
    assert e.value.code == _native.TSB_ERR_INVALID
    with pytest.raises(_native.TsbError, match=r"rect 0: a transposed rect has 2 to TSB_MAX_DIMS dims") as e:
        _native.transpose_compile_host(0, plain, 1)  # the plain copy collapses to one dim
    good = build_transpose_rects([(StridedMem(src.data_ptr(), (16, 8), (1, 16), torch.bfloat16, -1),
                                   StridedMem(dst.data_ptr(), (16, 8), (8, 1), torch.bfloat16, -1))])[0]
    arr = _native.make_rect_array(2)
    arr[0], arr[1] = good[0], good[0]
    arr[1].src_dtype, arr[1].dst_dtype = _native.TSB_F64, _native.TSB_BF16
    with pytest.raises(_native.TsbError, match=r"rect 1: no transposing kernel for dtype") as e:
        _native.transpose_compile_host(0, arr, 2)
    assert e.value.code == _native.TSB_ERR_UNSUPPORTED
    with pytest.raises(_native.TsbError, match=r"flags must be 0"):
        _native.transpose_compile_host(0, good, 1, flags=1)

"""GPU parity tests for direct_weight_sync.  The first block mirrors the reference's own tests
(tests/test_direct_weight_sync.py:103-276) with real NvlinkBuffer handles instead of the mock;
the second replays the golden plans recorded from the reference; the third checks a scaled
Llama-3 FSDP->TP sync against the numpy oracle."""

import itertools
import json
import os

import numpy as np
import pytest
import torch

from oracle import reshard_oracle as ro
from tests.helpers import DEV, llama_layout, run, sha256_of
from torchstore_b200.direct_weight_sync import (DirectWeightSyncDest, DirectWeightSyncSource, NvlinkBuffer,
                                                RDMAWeightHandle)
from torchstore_b200.transport.types import TensorSlice

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def _make_sharded_handles(original, num_shards, shard_dim, keep):
    handles = []
    shard_size = original.shape[shard_dim] // num_shards
    for rank in range(num_shards):
        idx = [slice(None)] * original.ndim
        idx[shard_dim] = slice(rank * shard_size, (rank + 1) * shard_size)
        shard = original[tuple(idx)].contiguous()
        keep.append(shard)
        offsets = [0] * original.ndim
        offsets[shard_dim] = rank * shard_size
        local_shape = list(original.shape)
        local_shape[shard_dim] = shard_size
        ts = TensorSlice(tuple(offsets), (rank,), tuple(original.shape), tuple(local_shape), (num_shards,))
        handles.append(RDMAWeightHandle(NvlinkBuffer(shard), ts, rank))
    return handles


def _make_replicated_handles(original, num_ranks, keep):
    handles = []
    for rank in range(num_ranks):
        data = original.clone()
        keep.append(data)
        ts = TensorSlice(tuple(0 for _ in original.shape), (rank,), tuple(original.shape), tuple(original.shape), (num_ranks,))
        handles.append(RDMAWeightHandle(NvlinkBuffer(data), ts, rank))
    return handles


def test_exact_match():
    keep = []
    original = torch.arange(512 * 512, dtype=torch.float32, device=DEV).reshape(512, 512)
    handles = _make_sharded_handles(original, 1, 0, keep)
    dest = torch.zeros_like(original)
    sync = DirectWeightSyncDest()
    run(sync.pull({"weight": handles}, {"weight": dest}))
    assert torch.equal(dest, original)
    assert len(sync._plan) == 1
    assert sync._plan[0].dest_tensor is None
    assert sync._plan[0].recv_buffer is None


@pytest.mark.parametrize("num_shards,shard_dim", [(2, 0), (4, 0), (2, 1)])
def test_resharding(num_shards, shard_dim):
    keep = []
    original = torch.arange(512 * 512, dtype=torch.float32, device=DEV).reshape(512, 512)
    handles = _make_sharded_handles(original, num_shards, shard_dim, keep)
    dest = torch.zeros_like(original)
    sync = DirectWeightSyncDest()
    run(sync.pull({"weight": handles}, {"weight": dest}))
    assert torch.equal(dest, original)
    assert len(sync._plan) == num_shards
    # no temporaries, unlike the reference's full-shard recv buffers
    assert all(op.recv_buffer is None for op in sync._plan)


def test_replicated_dedup():
    keep = []
    original = torch.arange(512 * 512, dtype=torch.float32, device=DEV).reshape(512, 512)
    handles = _make_replicated_handles(original, 2, keep)
    dest = torch.zeros_like(original)
    sync = DirectWeightSyncDest()
    run(sync.pull({"weight": handles}, {"weight": dest}))
    assert torch.equal(dest, original)
    assert len(sync._plan) == 1


def test_multiple_params():
    keep = []
    w1 = torch.arange(100, dtype=torch.float32, device=DEV).reshape(10, 10)
    w2 = torch.arange(100, 200, dtype=torch.float32, device=DEV).reshape(10, 10)
    all_handles = {
        "layer.weight": _make_sharded_handles(w1, 2, 0, keep),
        "layer.bias": _make_sharded_handles(w2, 1, 0, keep),
    }
    dest_sd = {"layer.weight": torch.zeros_like(w1), "layer.bias": torch.zeros_like(w2)}
    sync = DirectWeightSyncDest()
    run(sync.pull(all_handles, dest_sd))
    assert torch.equal(dest_sd["layer.weight"], w1)
    assert torch.equal(dest_sd["layer.bias"], w2)
    # one launch for the whole state dict
    assert len(sync._native_plans) == 1


def test_register_zero_copy_and_repeat_pull_sees_updates():
    """No transfer_dtype: handles point at live param memory, an in-place update is visible to the
    next pull without refresh (reference docstring :85-87)."""
    w = torch.arange(64 * 32, dtype=torch.float32, device=DEV).reshape(64, 32)
    source = DirectWeightSyncSource()
    handles = source.register({"w": w}, rank=0)
    assert source.refresh() == 0
    dest = torch.zeros_like(w)
    sync = DirectWeightSyncDest()
    all_handles = {"w": [handles["w"]]}
    run(sync.pull(all_handles, {"w": dest}))
    assert torch.equal(dest, w)
    w.mul_(2.0)
    run(sync.pull(all_handles, {"w": dest}))
    assert torch.equal(dest, w)
    run(source.cleanup())


def test_register_rejects_non_contiguous_without_transfer_dtype():
    backing = torch.arange(100, dtype=torch.float32, device=DEV).reshape(10, 10)
    with pytest.raises(AssertionError, match="Expected contiguous tensor"):
        DirectWeightSyncSource().register({"w": backing[:, :5]}, rank=0)


def test_refresh_with_staging_non_contiguous_source():
    """Non-contiguous param + transfer_dtype (same dtype): staging follows refresh()."""
    backing = torch.arange(100, dtype=torch.float32, device=DEV).reshape(10, 10)
    src = backing[:, :5]
    source = DirectWeightSyncSource()
    handles = source.register({"weight": src}, rank=0, transfer_dtype=torch.float32)
    assert "weight" in source._staging
    dest = torch.zeros(10, 5, dtype=torch.float32, device=DEV)
    run(DirectWeightSyncDest().pull({"weight": [handles["weight"]]}, {"weight": dest}))
    assert torch.equal(dest, src)
    backing.fill_(99.0)
    staging = source._staging["weight"][0]
    assert not torch.equal(staging, src)
    assert source.refresh() == 1
    assert torch.equal(staging, src)
    dest2 = torch.zeros(10, 5, dtype=torch.float32, device=DEV)
    run(DirectWeightSyncDest().pull({"weight": [handles["weight"]]}, {"weight": dest2}))
    assert torch.equal(dest2, torch.full((10, 5), 99.0, device=DEV))


def test_transfer_dtype():
    """fp32 master weights, bf16 transfer: dest equals original.to(bfloat16) bit for bit."""
    original = torch.arange(100, dtype=torch.float32, device=DEV).reshape(10, 10)
    source = DirectWeightSyncSource()
    handles = source.register({"weight": original}, rank=0, transfer_dtype=torch.bfloat16)
    dest = torch.zeros(10, 10, dtype=torch.bfloat16, device=DEV)
    run(DirectWeightSyncDest().pull({"weight": [handles["weight"]]}, {"weight": dest}))
    assert torch.equal(dest, original.to(torch.bfloat16))
    original.fill_(42.0)
    source.refresh()
    assert torch.equal(source._staging["weight"][0], torch.full((10, 10), 42.0, dtype=torch.bfloat16, device=DEV))
    dest2 = torch.zeros(10, 10, dtype=torch.bfloat16, device=DEV)
    run(DirectWeightSyncDest().pull({"weight": [handles["weight"]]}, {"weight": dest2}))
    assert torch.equal(dest2, torch.full((10, 10), 42.0, dtype=torch.bfloat16, device=DEV))


def test_cast_fused_into_gather_when_handle_dtype_differs():
    """Extension: source registered in fp32 (zero-copy), bf16 destination -> cast on read."""
    w = torch.randn(256, 384, device=DEV)
    handles = DirectWeightSyncSource().register({"w": w}, rank=0)
    dest = torch.zeros(256, 384, dtype=torch.bfloat16, device=DEV)
    run(DirectWeightSyncDest().pull({"w": [handles["w"]]}, {"w": dest}))
    assert torch.equal(dest, w.to(torch.bfloat16))


def test_nvlink_buffer_read_write_drop_and_pickle():
    import pickle

    from torchstore_b200.utils import to_byte_view

    src = torch.arange(4096, dtype=torch.int32, device=DEV)
    buf = pickle.loads(pickle.dumps(NvlinkBuffer(src)))
    out = torch.zeros_like(src)
    run(buf.read_into(to_byte_view(out)))
    assert torch.equal(out, src)
    new = torch.full_like(src, 5)
    run(buf.write_from(to_byte_view(new)))
    assert torch.equal(src, new)
    with pytest.raises(RuntimeError, match="size mismatch"):
        run(buf.read_into(to_byte_view(out[:10])))
    with pytest.raises(RuntimeError, match="CPU tensor"):
        run(buf.read_into(torch.zeros(4096 * 4, dtype=torch.uint8)))
    run(buf.drop())


def test_cpu_destination_fails_loudly():
    w = torch.randn(8, 8, device=DEV)
    handles = DirectWeightSyncSource().register({"w": w}, rank=0)
    with pytest.raises(RuntimeError, match="no CPU data path"):
        run(DirectWeightSyncDest().pull({"w": [handles["w"]]}, {"w": torch.zeros(8, 8)}))


# ---------------------------------------------------------------------------------------------
# golden plans from the reference
# ---------------------------------------------------------------------------------------------
def test_golden_reference_plans_and_results():
    cases = json.load(open(os.path.join(GOLDEN, "direct_plan.json")))["cases"]
    for case in cases:
        keep, all_handles, dest_sd, dest_slices = [], {}, {}, {}
        for name, p in case["params"].items():
            shape = tuple(p["global_shape"])
            full = (torch.arange(int(np.prod(shape)), dtype=torch.float32) + p["arange_start"]).reshape(shape).to(DEV)
            smesh = tuple(p["src_mesh"])
            spl = [tuple(x) for x in p["src_placements"]]
            hl = []
            for rank, coord in enumerate(itertools.product(*(range(m) for m in smesh))):
                sl = ro.make_slice(shape, smesh, coord, spl)
                shard = full[tuple(slice(o, o + s) for o, s in zip(sl.offsets, sl.local_shape))].contiguous()
                keep.append(shard)
                ts = TensorSlice(sl.offsets, sl.coordinates, sl.global_shape, sl.local_shape, sl.mesh_shape)
                hl.append(RDMAWeightHandle(NvlinkBuffer(shard), ts, rank))
            all_handles[name] = hl
            if p["dst_mesh"] is None:
                dest_sd[name] = torch.zeros(shape, dtype=torch.float32, device=DEV)
            else:
                dmesh = tuple(p["dst_mesh"])
                coord = list(itertools.product(*(range(m) for m in dmesh)))[p["dst_rank"]]
                dsl = ro.make_slice(shape, dmesh, coord, [tuple(x) for x in p["dst_placements"]])
                dest_sd[name] = torch.zeros(dsl.local_shape, dtype=torch.float32, device=DEV)
                dest_slices[name] = TensorSlice(dsl.offsets, dsl.coordinates, dsl.global_shape, dsl.local_shape, dsl.mesh_shape)
        sync = DirectWeightSyncDest()
        run(sync.pull(all_handles, dest_sd, dest_slices or None))
        index_of = {id(h.rdma_buffer): (n, i) for n, hl in all_handles.items() for i, h in enumerate(hl)}
        got_ops = []
        for op in sync._plan:
            n, i = index_of[id(op.rdma_buffer)]
            got_ops.append({
                "name": n, "source_index": i, "source_rank": all_handles[n][i].source_rank,
                "exact": op.dest_tensor is None,
                "src_index": None if op.src_slices is None else [[s.start, s.stop] for s in op.src_slices],
                "dest_index": None if op.dest_slices is None else [[s.start, s.stop] for s in op.dest_slices],
            })
        assert got_ops == case["ops"], case["label"]
        for name, digest in case["dest_sha256"].items():
            assert sha256_of(dest_sd[name]) == digest, (case["label"], name)
        sync.close()


# ---------------------------------------------------------------------------------------------
# scaled Llama-3 FSDP(n) -> TP(n), all ranks emulated on one GPU, against the numpy oracle
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2, 4, 8])
def test_scaled_llama_fsdp_to_tp_matches_oracle(n):
    layout = llama_layout(n_layers=2, scale=8)  # dims stay multiples of 8 ranks
    gen = torch.Generator().manual_seed(0)
    fulls = {k: (torch.randn(shape, generator=gen) * 0.02).to(torch.bfloat16) for k, (shape, _) in layout.items()}
    keep, all_handles, np_sources, np_handles = [], {}, {}, {}
    for name, (shape, _) in layout.items():
        hl, nps, nph = [], [], []
        for r in range(n):
            sl = ro.make_slice(shape, (n,), (r,), [("S", 0)])
            shard = fulls[name][tuple(slice(o, o + s) for o, s in zip(sl.offsets, sl.local_shape))].contiguous()
            dev_shard = shard.to(DEV)
            keep.append(dev_shard)
            ts = TensorSlice(sl.offsets, sl.coordinates, sl.global_shape, sl.local_shape, sl.mesh_shape)
            hl.append(RDMAWeightHandle(NvlinkBuffer(dev_shard), ts, r))
            nps.append(shard.view(torch.int16).numpy())
            nph.append((sl, r))
        all_handles[name], np_sources[name], np_handles[name] = hl, nps, nph
    for drank in range(n):
        dest_sd, dest_slices, np_dest, np_dslices = {}, {}, {}, {}
        for name, (shape, tp) in layout.items():
            dsl = ro.full_slice(shape) if n == 1 else ro.make_slice(shape, (n,), (drank,), [tp])
            dest_sd[name] = torch.zeros(dsl.local_shape, dtype=torch.bfloat16, device=DEV)
            if n > 1:
                dest_slices[name] = TensorSlice(dsl.offsets, dsl.coordinates, dsl.global_shape, dsl.local_shape, dsl.mesh_shape)
            np_dest[name] = np.zeros(dsl.local_shape, dtype=np.int16)
            np_dslices[name] = dsl
        sync = DirectWeightSyncDest()
        run(sync.pull(all_handles, dest_sd, dest_slices or None))
        plan = ro.build_plan(np_handles, np_dslices)
        assert len(plan) == len(sync._plan)
        ro.pull(plan, np_sources, np_dest)
        for name in layout:
            assert np.array_equal(dest_sd[name].cpu().view(torch.int16).numpy(), np_dest[name]), (n, drank, name)
        info = sync.plan_info()[0]
        assert info["payload_bytes"] == sum(v.numel() * 2 for v in dest_sd.values())
        assert info["src_bytes"] == info["payload_bytes"]  # no read amplification
        sync.close()


def test_plan_rebuilt_when_destination_changes():
    """A cached plan must never write tensors of a previous call (the reference's single cached plan
    would; see state_dict_utils.py:198-201)."""
    w = torch.randn(64, 64, device=DEV)
    handles = DirectWeightSyncSource().register({"w": w}, rank=0)
    sync = DirectWeightSyncDest()
    d1 = torch.zeros(64, 64, device=DEV)
    run(sync.pull({"w": [handles["w"]]}, {"w": d1}))
    d2 = torch.zeros(64, 64, device=DEV)
    run(sync.pull({"w": [handles["w"]]}, {"w": d2}))
    assert torch.equal(d1, w) and torch.equal(d2, w)


def test_same_dict_pull_launches_first_and_still_catches_in_place_edits():
    """Passing the very dict object of the last pull launches the cached plan before validating it; an
    edit of that dict in between (a value replaced, or a tensor's storage swapped under the same object)
    is caught while the kernel runs and the pull is redone into the right memory."""
    w = torch.randn(256, 128, device=DEV)
    b = torch.randn(128, device=DEV)
    handles = DirectWeightSyncSource().register({"w": w, "b": b}, rank=0)
    hs = {"w": [handles["w"]], "b": [handles["b"]]}
    dest = {"w": torch.zeros(256, 128, device=DEV), "b": torch.zeros(128, device=DEV)}
    sync = DirectWeightSyncDest()
    run(sync.pull(hs, dest))
    plan0 = dict(sync._native_plans)
    w.add_(1.0)
    torch.cuda.synchronize()
    run(sync.pull(hs, dest))                      # same dict object, nothing edited: cached plan replayed
    assert sync._native_plans == plan0 and torch.equal(dest["w"], w)
    old_w = dest["w"]
    dest["w"] = torch.zeros(256, 128, device=DEV)  # value replaced inside the same dict
    run(sync.pull(hs, dest))
    assert torch.equal(dest["w"], w) and sync._native_plans != plan0
    assert torch.equal(old_w, w)                   # the speculative launch filled the old tensor: harmless
    plan1 = dict(sync._native_plans)
    dest["b"].data = torch.zeros(128, device=DEV)  # same object, other storage
    b.mul_(3.0)
    torch.cuda.synchronize()
    run(sync.pull(hs, dest))
    assert torch.equal(dest["b"], b) and sync._native_plans != plan1
    sync.close()

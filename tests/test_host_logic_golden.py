"""The product's own index math (torchstore_b200/utils.py, transport/types.py, the direct-sync
planner) against the fixtures recorded from the reference.  CPU only: plans are built on host
tensors and checked as metadata; bytes are moved by the ORACLE's C routine from the product's
rectangle descriptors, which validates planner + descriptor builder end to end without a GPU."""

import itertools
import json
import os

import numpy as np
import pytest
import torch

from oracle import c_oracle
from oracle import reshard_oracle as ro
from tests.helpers import HostBuffer, sha256_of
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, RDMAWeightHandle
from torchstore_b200.planner import StridedMem, build_rects
from torchstore_b200.transport.types import Request, TensorSlice
from torchstore_b200.utils import (assemble_tensor, get_destination_region, get_destination_view, get_local_tensor,
                                   get_slice_intersection, to_byte_view)

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def load(name):
    with open(os.path.join(GOLDEN, name)) as f:
        return json.load(f)


def TS(j):
    if j is None:
        return None
    return TensorSlice(tuple(j["offsets"]), None if j["coordinates"] is None else tuple(j["coordinates"]),
                       tuple(j["global_shape"]), tuple(j["local_shape"]),
                       None if j["mesh_shape"] is None else tuple(j["mesh_shape"]))


def test_get_slice_intersection_golden():
    for c in load("slice_math.json")["intersections"]:
        got = get_slice_intersection(TS(c["stored"]), TS(c["wanted"]))
        want = TS(c["result"])
        assert (got is None) == (want is None), c
        if want is not None:
            assert got == want, c


def test_get_destination_view_golden():
    for c in load("slice_math.json")["dest_views"]:
        shape = tuple(c["dest_shape"])
        if c["dest_contiguous"]:
            dest = torch.zeros(shape)
        else:
            dest = torch.zeros(tuple(reversed(shape))).permute(*reversed(range(len(shape))))
        view = get_destination_view(dest, TS(c["dest_slice"]), TS(c["fetch"]))
        if c["result"] is None:
            assert view is None, c
        else:
            assert view is not None, c
            idx = tuple(slice(a, b) for a, b in c["result"])
            assert view.data_ptr() == dest[idx].data_ptr() and tuple(view.shape) == tuple(dest[idx].shape), c
            # the strided variant agrees wherever the contiguous rule accepts
            region = get_destination_region(dest, TS(c["dest_slice"]), TS(c["fetch"]))
            assert region.data_ptr() == view.data_ptr() and region.shape == view.shape


def test_assemble_and_local_tensor_golden():
    d = load("slice_math.json")
    for c in d["assemble"]:
        got = assemble_tensor([torch.tensor(p) for p in c["parts"]], [tuple(o) for o in c["offsets"]])
        assert got.tolist() == c["result"], c
    for c in d["get_local_tensor"]:
        assert get_local_tensor(torch.tensor(c["global"]), tuple(c["shape"]), tuple(c["offset"])).tolist() == c["result"]
    with pytest.raises(AssertionError):
        assemble_tensor([], [])
    with pytest.raises(AssertionError):  # gap: parts cannot fill the bounding box
        assemble_tensor([torch.tensor([1]), torch.tensor([2])], [(0,), (5,)])


def test_to_byte_view():
    assert to_byte_view(torch.tensor(1.5)).shape == (4,)
    t = torch.arange(6, dtype=torch.int16).reshape(2, 3)
    assert to_byte_view(t).shape == (12,) and to_byte_view(t).data_ptr() == t.data_ptr()


def test_direct_plan_golden_ops_and_bytes_via_oracle_executor():
    cases = load("direct_plan.json")["cases"]
    for case in cases:
        all_handles, dest_sd, dest_slices = {}, {}, {}
        for name, p in case["params"].items():
            shape = tuple(p["global_shape"])
            full = (torch.arange(int(np.prod(shape)), dtype=torch.float32) + p["arange_start"]).reshape(shape)
            smesh = tuple(p["src_mesh"])
            spl = [tuple(x) for x in p["src_placements"]]
            hl = []
            for rank, coord in enumerate(itertools.product(*(range(m) for m in smesh))):
                sl = ro.make_slice(shape, smesh, coord, spl)
                shard = full[tuple(slice(o, o + s) for o, s in zip(sl.offsets, sl.local_shape))].contiguous()
                ts = TensorSlice(sl.offsets, sl.coordinates, sl.global_shape, sl.local_shape, sl.mesh_shape)
                hl.append(RDMAWeightHandle(HostBuffer(shard, shard.shape, shard.dtype), ts, rank))
            all_handles[name] = hl
            if p["dst_mesh"] is None:
                dest_sd[name] = torch.zeros(shape)
            else:
                dmesh = tuple(p["dst_mesh"])
                coord = list(itertools.product(*(range(m) for m in dmesh)))[p["dst_rank"]]
                dsl = ro.make_slice(shape, dmesh, coord, [tuple(x) for x in p["dst_placements"]])
                dest_sd[name] = torch.zeros(dsl.local_shape)
                dest_slices[name] = TensorSlice(dsl.offsets, dsl.coordinates, dsl.global_shape, dsl.local_shape, dsl.mesh_shape)
        sync = DirectWeightSyncDest()
        plan = sync._build_plan(all_handles, dest_sd, dest_slices or None)
        index_of = {id(h.rdma_buffer): (n, i) for n, hl in all_handles.items() for i, h in enumerate(hl)}
        got = []
        for op in plan:
            n, i = index_of[id(op.rdma_buffer)]
            got.append({"name": n, "source_index": i, "source_rank": all_handles[n][i].source_rank,
                        "exact": op.dest_tensor is None,
                        "src_index": None if op.src_slices is None else [[s.start, s.stop] for s in op.src_slices],
                        "dest_index": None if op.dest_slices is None else [[s.start, s.stop] for s in op.dest_slices]})
        assert got == case["ops"], case["label"]
        # descriptors built by the product, bytes moved by the oracle
        pairs = [sync.op_windows(op, StridedMem.from_tensor(op.rdma_buffer.shard)) for op in plan]
        rects, n = build_rects(pairs)
        c_oracle.copy_rects(rects, n)
        for name, digest in case["dest_sha256"].items():
            assert sha256_of(dest_sd[name]) == digest, (case["label"], name)


def test_request_from_dtensor_on_fake_process_group():
    """DTensor -> (local tensor alias, TensorSlice) exactly as torch computes the layout."""
    import torch.distributed as dist
    from torch.distributed.device_mesh import DeviceMesh
    from torch.distributed.tensor import DTensor, Replicate, Shard
    from torch.testing._internal.distributed.fake_pg import FakeStore

    for rank in (0, 5):
        dist.init_process_group("fake", store=FakeStore(), rank=rank, world_size=8)
        try:
            mesh = DeviceMesh("cpu", torch.arange(8).reshape(2, 4))
            full = torch.arange(64 * 32, dtype=torch.float32).reshape(64, 32)
            coord = mesh.get_coordinate()
            want = ro.make_slice((64, 32), (2, 4), tuple(coord), [("S", 0), ("S", 1)])
            local = full[tuple(slice(o, o + s) for o, s in zip(want.offsets, want.local_shape))].contiguous()
            dt = DTensor.from_local(local, mesh, (Shard(0), Shard(1)), run_check=False, shape=full.shape, stride=full.stride())
            req = Request.from_any("w", dt)
            assert req.tensor_val.data_ptr() == local.data_ptr()
            assert tuple(req.tensor_slice.offsets) == want.offsets and tuple(req.tensor_slice.local_shape) == want.local_shape
            assert tuple(req.tensor_slice.coordinates) == tuple(coord) and tuple(req.tensor_slice.mesh_shape) == (2, 4)
            with pytest.raises(ValueError, match="Cannot specify tensor_slice with a DTensor"):
                Request.from_any("w", dt, req.tensor_slice)
            # fully replicated DTensor is stored as a plain tensor
            rep = DTensor.from_local(full, mesh, (Replicate(), Replicate()), run_check=False)
            r2 = Request.from_any("w", rep)
            assert r2.tensor_slice is None and r2.tensor_val.data_ptr() == full.data_ptr()
        finally:
            dist.destroy_process_group()

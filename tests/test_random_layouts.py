"""Seeded random DeviceMesh/placement pairs: the product's direct-sync planner + rectangle builder
(bytes moved by the oracle's C executor on host memory) must reproduce, for every destination rank,
exactly the slice of the global tensor that rank owns -- and agree op-for-op with the numpy oracle's
restatement of the reference planner.  Covers uneven and empty shards, 2-D meshes, replication on
either side and 1-3-D tensors (the reference tests only 1-D/2-D even layouts)."""

import itertools
import random

import numpy as np
import pytest
import torch

from oracle import c_oracle
from oracle import reshard_oracle as ro
from tests.helpers import HostBuffer
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, RDMAWeightHandle
from torchstore_b200.planner import StridedMem, build_rects
from torchstore_b200.transport.types import TensorSlice


def rand_layout(rng, ndim):
    md = rng.choice([1, 1, 2])
    mesh = tuple(rng.choice([1, 2, 3, 4]) for _ in range(md))
    pl = [rng.choice([("R",)] + [("S", d) for d in range(ndim)]) for _ in range(md)]
    return mesh, pl


def to_ts(sl):
    return TensorSlice(sl.offsets, sl.coordinates, sl.global_shape, sl.local_shape, sl.mesh_shape)


@pytest.mark.parametrize("seed", range(6))
def test_random_mesh_pairs(seed):
    rng = random.Random(4242 + seed)
    for _ in range(25):
        ndim = rng.choice([1, 2, 2, 3])
        shape = tuple(rng.choice([1, 3, 4, 6, 7, 8, 12, 16, 17]) for _ in range(ndim))
        dtype = rng.choice([torch.float32, torch.bfloat16, torch.int64, torch.uint8])
        full = torch.arange(int(np.prod(shape))).reshape(shape).to(dtype)
        smesh, spl = rand_layout(rng, ndim)
        dmesh, dpl = rand_layout(rng, ndim)
        handles, np_handles = [], []
        for rank, coord in enumerate(itertools.product(*(range(m) for m in smesh))):
            sl = ro.make_slice(shape, smesh, coord, spl)
            shard = full[tuple(slice(o, o + s) for o, s in zip(sl.offsets, sl.local_shape))].contiguous()
            handles.append(RDMAWeightHandle(HostBuffer(shard, shard.shape, shard.dtype), to_ts(sl), rank))
            np_handles.append((sl, rank))
        for coord in itertools.product(*(range(m) for m in dmesh)):
            dsl = ro.make_slice(shape, dmesh, coord, dpl)
            dest = torch.full(dsl.local_shape, -1 if dtype != torch.uint8 else 255).to(dtype)
            sync = DirectWeightSyncDest()
            plan = sync._build_plan({"w": handles}, {"w": dest}, {"w": to_ts(dsl)})
            oracle_plan = ro.build_plan({"w": np_handles}, {"w": dsl})
            assert len(plan) == len(oracle_plan)
            for op, oop in zip(plan, oracle_plan):
                assert (op.dest_tensor is None) == oop.exact
                assert op.src_slices == oop.src_index and op.dest_slices == oop.dest_index
            pairs = [sync.op_windows(op, StridedMem.from_tensor(op.rdma_buffer.shard)) for op in plan]
            rects, n = build_rects(pairs)
            c_oracle.copy_rects(rects, n)
            want = full[tuple(slice(o, o + s) for o, s in zip(dsl.offsets, dsl.local_shape))]
            assert torch.equal(dest, want), (shape, smesh, spl, dmesh, dpl, coord)

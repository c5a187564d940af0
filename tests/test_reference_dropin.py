"""Drop-in proof: our ``NvlinkBuffer`` handles went through the reference's UNMODIFIED
``DirectWeightSyncDest._build_plan`` (metadata only -- torchstore/direct_weight_sync.py:221-317), and
the op list it built (recorded by ``oracle/gen_golden.py`` in ``tests/golden/reference_dropin.json``)
must equal the one our own ``_build_plan`` builds from the same handles: same length, same order,
same exact/partial classification, same source/destination slices, same source per op.

Also checks the other half of the duck-type contract (direct_weight_sync.py:46-58): an
``RDMAWeightHandle`` carrying an ``NvlinkBuffer`` has the reference's fields, survives the pickle
round trip every store put performs, and exposes the coroutine methods the reference calls
(read_into / write_from / drop).
"""

import inspect
import json
import os
import pickle

import pytest
import torch

import workloads
from oracle.gen_golden import DROPIN_CASES, dropin_case_id
from torchstore_b200 import direct_weight_sync as ours
from torchstore_b200.planner import HbmDescriptor
from torchstore_b200.transport.types import TensorSlice as OurSlice

GOLDEN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_dropin.json")))


def _fake_buffer(shape, dtype, device):
    """An NvlinkBuffer as a destination process sees it after unpickling: descriptor only."""
    stride = []
    s = 1
    for e in reversed(shape):
        stride.append(s)
        s *= e
    desc = HbmDescriptor(region=bytes(120), shape=tuple(shape), stride=tuple(reversed(stride)), dtype=dtype, device=device)
    return ours.NvlinkBuffer(descriptor=desc)


def _slice(cls, shape, n, r, placement):
    off, shp = workloads.shard_box(shape, n, r, placement) if placement[0] == "S" else ((0,) * len(shape), tuple(shape))
    return cls(offsets=tuple(off), coordinates=(r,), global_shape=tuple(shape), local_shape=tuple(shp), mesh_shape=(n,))


def test_every_case_was_recorded():
    assert sorted(GOLDEN["cases"]) == sorted(dropin_case_id(c) for c in DROPIN_CASES)


@pytest.mark.parametrize("case", DROPIN_CASES, ids=lambda c: f"{c[0]}-{c[1]}{c[2]}->{c[3]}{c[4]}")
def test_reference_build_plan_accepts_nvlink_buffers_and_matches_ours(case):
    shape, n_src, sp, n_dst, dp = case
    recorded = GOLDEN["cases"][dropin_case_id(case)]
    checked = 0
    for drank in range(n_dst):
        our_handles, rank_of = [], {}
        for r in range(n_src):
            rs = _slice(OurSlice, shape, n_src, r, sp)
            if 0 in rs.local_shape:
                continue
            buf = _fake_buffer(rs.local_shape, torch.float32, r)
            rank_of[id(buf)] = r
            our_handles.append(ours.RDMAWeightHandle(rdma_buffer=buf, tensor_slice=rs, source_rank=r))
        ds_our = _slice(OurSlice, shape, n_dst, drank, dp)
        if 0 in ds_our.local_shape:
            assert str(drank) not in recorded
            continue
        dest = torch.zeros(ds_our.local_shape, dtype=torch.float32)
        ref_ops = recorded[str(drank)]
        our_ops = ours.DirectWeightSyncDest()._build_plan({"w": our_handles}, {"w": dest}, {"w": ds_our})
        assert len(ref_ops) == len(our_ops) > 0
        for a, b in zip(ref_ops, our_ops):
            assert a["source_rank"] == rank_of[id(b.rdma_buffer)]  # same source, same order
            assert a["exact"] == (b.dest_tensor is None)
            if not a["exact"]:
                assert tuple(slice(*s) for s in a["src_slices"]) == tuple(b.src_slices)
                assert tuple(slice(*s) for s in a["dest_slices"]) == tuple(b.dest_slices)
                assert b.dest_tensor is dest
                # the reference stages the WHOLE source shard; we describe just the overlap rectangle
                assert tuple(a["recv_shape"]) == tuple(b.rdma_buffer.shape)
            else:
                assert b.dest_byte_view.data_ptr() == dest.data_ptr()
        checked += 1
    assert checked == len(recorded)


def test_handle_pickles_and_duck_types_like_an_rdma_buffer():
    import dataclasses

    assert [f.name for f in dataclasses.fields(ours.RDMAWeightHandle)] == GOLDEN["handle_fields"]
    buf = _fake_buffer((16, 8), torch.bfloat16, 3)
    h = ours.RDMAWeightHandle(rdma_buffer=buf, tensor_slice=_slice(OurSlice, (32, 8), 2, 1, ("S", 0)), source_rank=1)
    h2 = pickle.loads(pickle.dumps(h))
    assert h2.rdma_buffer.descriptor == buf.descriptor and h2.tensor_slice == h.tensor_slice and h2.source_rank == 1
    assert h2.rdma_buffer.nbytes == 16 * 8 * 2 and h2.rdma_buffer.dtype == torch.bfloat16
    assert set(GOLDEN["buffer_methods_called"]) <= {"read_into", "write_from", "drop"}
    for name in ("read_into", "write_from", "drop"):  # call sites direct_weight_sync.py:143,174,339
        assert inspect.iscoroutinefunction(getattr(h2.rdma_buffer, name))
    # CPU tensors are refused loudly (no host data plane behind this handle)
    import asyncio

    with pytest.raises(RuntimeError):
        asyncio.run(h2.rdma_buffer.read_into(torch.zeros(16 * 8 * 2, dtype=torch.uint8)))

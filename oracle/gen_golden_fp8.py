"""TEST INFRASTRUCTURE ONLY -- generate the fp8 fixtures of tests/golden/ from torch and the UNMODIFIED
reference (run on its own, where the reference tree is present, TORCHSTORE_REFERENCE_ROOT):
    python oracle/gen_golden_fp8.py [fp8_cast_vectors] [direct_fp8]      (no argument: both)
The outputs are committed; nothing under tests/ reads the reference at run time.

  fp8_cast_vectors.npz  torch CPU .to() bit patterns for the fp8 pairs: every bf16 and f16 pattern and
                      an f32 edge/boundary/random set -> float8_e4m3fn and float8_e5m2, every pattern
                      of both fp8 formats -> f32, bf16 and f16
  direct_fp8.json     DirectWeightSyncDest.pull of FSDP -> TP layouts into fp8 destinations, sources
                      staged with the reference's own register() staging, local.to(fp8) (sha256)

The helpers shared with the other fixtures (MockRDMABuffer, sha, the f32 edge set of cast_vectors.npz)
come from oracle/gen_golden.py.
"""

from __future__ import annotations

import asyncio
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import ref_harness  # noqa: E402
from oracle.gen_golden import GOLDEN, MockRDMABuffer, gen_cast_vectors, sha  # noqa: E402

FP8_DTYPES = {"float8_e4m3fn": torch.float8_e4m3fn, "float8_e5m2": torch.float8_e5m2}


def gen_fp8_cast_vectors():
    rng = np.random.default_rng(8)
    base = gen_cast_vectors()["f32"][:35]  # the f32 edge set of gen_cast_vectors
    bounds = np.array([448.0, 464.0, 480.0, 57344.0, 61440.0, 2.0 ** -9, 2.0 ** -10, 2.0 ** -6, 2.0 ** -14,
                       2.0 ** -16, 2.0 ** -17, 65536.0, 496.0, 448.0 + 8.0, 59392.0], dtype=np.float32).view(np.uint32)
    ulp = np.concatenate([bounds - 1, bounds + 1])  # one f32 ulp either side of every boundary
    specials = np.array([0x7F800000, 0x7FC00000, 0x7F800001, 0x7FFFFFFF], dtype=np.uint32)  # +Inf, NaNs
    edge = np.concatenate([bounds, ulp, specials])
    edge = np.concatenate([edge, edge | np.uint32(0x80000000)])  # both signs
    rnd = rng.integers(0, 2**32, size=8192, dtype=np.uint64).astype(np.uint32)
    # magnitudes over the whole fp8 range (subnormals to overflow), random sign
    mag = (2.0 ** rng.uniform(-20, 18, size=8192)).astype(np.float32).view(np.uint32)
    mag |= (rng.integers(0, 2, size=8192).astype(np.uint32) << np.uint32(31))
    f32 = np.concatenate([base, edge, rnd, mag])
    out = {"f32": f32}
    t32 = torch.from_numpy(f32.view(np.float32).copy())
    all16 = np.arange(0, 65536, dtype=np.uint32).astype(np.uint16)
    out["all16"] = all16
    srcs = {"f32": t32,
            "bf16": torch.from_numpy(all16.view(np.int16).copy()).view(torch.bfloat16),
            "f16": torch.from_numpy(all16.view(np.int16).copy()).view(torch.float16)}
    short = {"float8_e4m3fn": "e4m3", "float8_e5m2": "e5m2"}
    for sname, t in srcs.items():
        for fname, fdt in FP8_DTYPES.items():
            out[f"{sname}_to_{short[fname]}"] = t.to(fdt).view(torch.uint8).numpy().copy()
    all8 = np.arange(0, 256, dtype=np.uint32).astype(np.uint8)
    out["all8"] = all8
    for fname, fdt in FP8_DTYPES.items():
        t8 = torch.from_numpy(all8.copy()).view(fdt)
        out[f"{short[fname]}_to_f32"] = t8.to(torch.float32).view(torch.int32).numpy().view(np.uint32)
        out[f"{short[fname]}_to_bf16"] = t8.to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
        out[f"{short[fname]}_to_f16"] = t8.to(torch.float16).view(torch.int16).numpy().view(np.uint16)
    return out


# (global shape, source dtype, transfer dtype, n FSDP source ranks, n TP destination ranks, TP placement)
DIRECT_FP8_CASES = [
    ((256, 192), "bfloat16", "float8_e4m3fn", 4, 2, ("S", 1)),
    ((256, 192), "bfloat16", "float8_e5m2", 4, 4, ("S", 0)),
    ((96, 80), "float32", "float8_e4m3fn", 2, 4, ("S", 1)),
    ((96, 80), "float32", "float8_e5m2", 8, 2, ("S", 1)),
    ((50, 48), "bfloat16", "float8_e4m3fn", 4, 3, ("S", 1)),  # uneven
    ((64, 32), "float32", "float8_e4m3fn", 2, 2, ("R",)),
]


def direct_fp8_full(gshape, src_dtype, seed):
    """The global tensor of a direct_fp8 case: normal values spread over the fp8 range, with a few
    entries past its largest finite values, so the saturation rules are reached."""
    g = torch.Generator().manual_seed(seed)
    full = torch.randn(gshape, generator=g) * 2.0 ** torch.randint(-12, 12, gshape, generator=g).float()
    full.view(-1)[::97] *= 7e4
    return full.to(getattr(torch, src_dtype))


def gen_direct_fp8():
    """The reference's DirectWeightSyncDest.pull into fp8 destinations; every source shard is staged
    the way the reference's register(transfer_dtype=fp8) stages it (local_tensor.to(transfer_dtype))
    and read through MockRDMABuffer (tests/test_direct_weight_sync.py:27-37)."""
    import torchstore.direct_weight_sync as ref
    from torchstore.transport.types import TensorSlice as RefSlice
    from torchstore.utils import to_byte_view

    import workloads

    def mk_slice(shape, n, r, placement):
        off, shp = workloads.shard_box(shape, n, r, placement) if placement[0] == "S" else ((0,) * len(shape), tuple(shape))
        return RefSlice(offsets=tuple(off), coordinates=(r,), global_shape=tuple(shape), local_shape=tuple(shp), mesh_shape=(n,))

    cases = []
    saved = ref._request_to_slice
    try:
        for i, (gshape, sdt, tdt, n_src, n_dst, dp) in enumerate(DIRECT_FP8_CASES):
            full = direct_fp8_full(gshape, sdt, seed=100 + i)
            fdt = FP8_DTYPES[tdt]
            handles = []
            for r in range(n_src):
                rs = mk_slice(gshape, n_src, r, ("S", 0))
                if 0 in rs.local_shape:
                    continue
                local = full[tuple(slice(o, o + s) for o, s in zip(rs.offsets, rs.local_shape))]
                staged = local.to(fdt).contiguous()  # reference direct_weight_sync.py:133
                handles.append(ref.RDMAWeightHandle(rdma_buffer=MockRDMABuffer(to_byte_view(staged)), tensor_slice=rs,
                                                    source_rank=r))
            per_rank = {}
            for drank in range(n_dst):
                ds = mk_slice(gshape, n_dst, drank, dp)
                if 0 in ds.local_shape:
                    continue
                dest = torch.zeros(ds.local_shape, dtype=fdt)
                ref._request_to_slice = lambda req, param, _s=ds: _s
                asyncio.run(ref.DirectWeightSyncDest().pull({"w": handles}, {"w": dest}))
                want = full.to(fdt)[tuple(slice(o, o + s) for o, s in zip(ds.offsets, ds.local_shape))]
                assert torch.equal(dest.view(torch.uint8), want.view(torch.uint8)), (gshape, sdt, tdt, drank)
                per_rank[str(drank)] = {"offsets": list(ds.offsets), "local_shape": list(ds.local_shape), "sha256": sha(dest)}
            cases.append({"global_shape": list(gshape), "src_dtype": sdt, "transfer_dtype": tdt, "seed": 100 + i,
                          "n_src": n_src, "src_placement": ["S", 0], "n_dst": n_dst, "dst_placement": list(dp),
                          "dest": per_rank})
    finally:
        ref._request_to_slice = saved
    return {"cases": cases}


def main(only=None):
    ref_harness.import_reference()
    os.makedirs(GOLDEN, exist_ok=True)
    if not only or "direct_fp8" in only:
        data = gen_direct_fp8()
        data["_meta"] = {"reference_commit": "ed2ddb67", "torch": torch.__version__, "generator": "oracle/gen_golden_fp8.py"}
        with open(os.path.join(GOLDEN, "direct_fp8.json"), "w") as f:
            json.dump(data, f, separators=(",", ":"))
        print("direct_fp8", os.path.getsize(os.path.join(GOLDEN, "direct_fp8.json")), "bytes")
    if not only or "fp8_cast_vectors" in only:
        np.savez_compressed(os.path.join(GOLDEN, "fp8_cast_vectors.npz"), **gen_fp8_cast_vectors())
        print("fp8_cast_vectors", os.path.getsize(os.path.join(GOLDEN, "fp8_cast_vectors.npz")), "bytes")


if __name__ == "__main__":
    main(sys.argv[1:] or None)

"""Source-side quantisation on one GPU: the Llama-3-8B linear weights (wq wk wv wo w1 w2 w3) in bf16, refreshed
into block-, channel- and tensor-scaled fp8 staging by DirectWeightSyncSource(quantize=...), alternated in the
same run with the plain bf16 -> e4m3fn staging refresh (transfer_dtype, KIND_BF16_E4M3) and with the existing
destination-side block and scaled pulls of the same weights from local bf16 handles.  A second phase refreshes
an FSDP(8)-style shard set of the same weights whose row boundaries sit 37 rows past multiples of N/8, so most
shards start mid-block and the shard-local anchoring runs at size.  A third phase refreshes the same weights held
in f32 (an fp32-master trainer) into block-scaled staging, beside the destination-side block pull from f32 handles.

    python tools/source_quant_bench.py [--reps 10] [--warmup 3]

Kernel times come from the plans' own start/done events, medians over warmed, repeated launches.  Bytes are
computed from the shapes: a refresh reads 2 bytes per element (twice per tensor: its pass 1 only folds the amax)
and writes 1 byte per element plus 4 per scale.  Alongside: the card's name and power limit and its measured
device-to-device copy rate (torch copy_ of 4 GiB), the ceiling the rates are compared with.  Every staging
buffer is checked bit for bit against the torch-CUDA rendering of the formula (source_quant_oracle.torch_quantize).
Prints one JSON line.
"""

import argparse
import asyncio
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import workloads  # noqa: E402
from oracle.source_quant_oracle import torch_quantize  # noqa: E402
from tools.fp8_sync_bench import copy_rate, entry  # noqa: E402
from torchstore_b200 import _native  # noqa: E402
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource  # noqa: E402
from torchstore_b200.transport.types import TensorSlice  # noqa: E402

E4M3 = torch.float8_e4m3fn
LINEAR = {"wq", "wk", "wv", "wo", "w1", "w2", "w3"}
GRANS = ("block", "channel", "tensor")
KW = {"block": "block_scales", "channel": "channel_scales", "tensor": "tensor_scales"}


def scale_like(gran: str, shape) -> torch.Tensor:
    if gran == "block":
        return torch.empty(-(-shape[0] // 128), -(-shape[1] // 128), device="cuda")
    if gran == "channel":
        return torch.empty(shape[0], 1, device="cuda")
    return torch.empty((), device="cuda")


def refresh_ms(src: DirectWeightSyncSource, plans) -> float:
    src.refresh()
    return plans.elapsed_ms()[0]


def exact(src: DirectWeightSyncSource, offsets: dict) -> bool:
    ok = True
    for name, (fp8, scale, local) in src._quantized.items():
        g = src._handles[name].rdma_buffer.granularity
        q, s = torch_quantize(local, g, *offsets.get(name, (0, 0)))
        ok &= torch.equal(fp8.view(torch.uint8), q.view(torch.uint8))
        ok &= torch.equal(scale.view(torch.int32), s.reshape(scale.shape).view(torch.int32))
        del q, s
    return bool(ok)


def fsdp_shards(sd: dict) -> tuple[dict, dict, dict]:
    """8 row shards per weight, views of the full tensors, boundaries at i * N / 8 + 37 (i = 1..7)."""
    shards, slices, offsets = {}, {}, {}
    for k, w in sd.items():
        n, c = w.shape
        cuts = [0] + [i * n // 8 + 37 for i in range(1, 8)] + [n]
        for r in range(8):
            r0, r1 = cuts[r], cuts[r + 1]
            name = f"{k}#{r}"
            shards[name] = w[r0:r1]
            slices[name] = TensorSlice((r0, 0), (r,), (n, c), (r1 - r0, c), (8,))
            offsets[name] = (r0, 0)
    return shards, slices, offsets


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    _native.init()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    copy_gbps = copy_rate(20)
    out = {"gpu": gpu, "copy_GBps_read_plus_write": round(copy_gbps, 1)}

    g = torch.Generator(device="cuda").manual_seed(0)
    layout = workloads.llama_layout()
    names = [k for k in layout if k.split(".")[-2] in LINEAR]
    sd = {k: (torch.randn(layout[k][0], device="cuda", generator=g) * 0.02).to(torch.bfloat16) for k in names}
    n = sum(v.numel() for v in sd.values())
    n_scales = {gran: sum(scale_like(gran, v.shape).numel() for v in sd.values()) for gran in GRANS}
    out["params"] = n

    def written(gran):
        return n + 4 * n_scales[gran]

    # phase 1: one full-size source per granularity, the plain cast refresh and the destination-side pulls
    srcs = {gran: DirectWeightSyncSource() for gran in GRANS}
    for gran, src in srcs.items():
        src.register(sd, rank=0, quantize={k: gran for k in sd})
    cast = DirectWeightSyncSource()
    cast.register(sd, rank=0, transfer_dtype=E4M3)
    trainer = DirectWeightSyncSource()
    handles = {k: [h] for k, h in trainer.register(sd, rank=0).items()}
    dest = {k: torch.empty(v.shape, dtype=E4M3, device="cuda") for k, v in sd.items()}
    dest_scales = {gran: {k: scale_like(gran, v.shape) for k, v in sd.items()} for gran in GRANS}
    pulls = {gran: DirectWeightSyncDest() for gran in GRANS}
    times = {k: [] for k in [f"{gran}_source_refresh" for gran in GRANS] + ["bf16_e4m3_cast_refresh"] +
             [f"{gran}_dest_side_pull" for gran in GRANS]}
    for i in range(args.warmup + args.reps):  # alternate every route
        t = {f"{gran}_source_refresh": refresh_ms(src, src._quant_plans) for gran, src in srcs.items()}
        t["bf16_e4m3_cast_refresh"] = refresh_ms(cast, cast._refresh_plans)
        for gran, sync in pulls.items():
            asyncio.run(sync.pull(handles, dest, **{KW[gran]: dest_scales[gran]}))
            t[f"{gran}_dest_side_pull"] = sync.last_pull_ms[0]
        if i >= args.warmup:
            for k, v in t.items():
                times[k].append(v)
    med = {k: statistics.median(v) for k, v in times.items()}
    for gran in GRANS:
        read = (4 if gran == "tensor" else 2) * n
        for form in ("source_refresh", "dest_side_pull"):
            out[f"{gran}_{form}"] = entry(med[f"{gran}_{form}"], read, written(gran), copy_gbps)
        out[f"{gran}_source_refresh"]["vs_dest_side_pull"] = round(med[f"{gran}_dest_side_pull"] / med[f"{gran}_source_refresh"], 3)
    out["bf16_e4m3_cast_refresh"] = entry(med["bf16_e4m3_cast_refresh"], 2 * n, n, copy_gbps)
    bit_exact = {f"full_{gran}": exact(src, {}) for gran, src in srcs.items()}
    for sync in pulls.values():
        sync.close()
    for src in list(srcs.values()) + [cast, trainer]:
        asyncio.run(src.cleanup())
    del srcs, cast, trainer, handles, dest, dest_scales
    torch.cuda.empty_cache()

    # phase 2: the FSDP(8)-style shard set, one source per granularity holding all 8 shards of every weight
    shards, slices, offsets = fsdp_shards(sd)
    srcs = {gran: DirectWeightSyncSource() for gran in GRANS}
    for gran, src in srcs.items():
        src.register(shards, rank=0, tensor_slices=slices, quantize={k: gran for k in shards})
    times = {gran: [] for gran in GRANS}
    for i in range(args.warmup + args.reps):
        for gran, src in srcs.items():
            ms = refresh_ms(src, src._quant_plans)
            if i >= args.warmup:
                times[gran].append(ms)
    for gran in GRANS:
        n_s = sum(s.numel() for _, s, _ in srcs[gran]._quantized.values())
        out[f"{gran}_source_refresh_fsdp8_unaligned"] = entry(statistics.median(times[gran]),
                                                              (4 if gran == "tensor" else 2) * n, n + 4 * n_s, copy_gbps)
        bit_exact[f"fsdp8_{gran}"] = exact(srcs[gran], offsets)
    for src in srcs.values():
        asyncio.run(src.cleanup())
    del srcs, shards
    torch.cuda.empty_cache()

    # phase 3: an fp32-master trainer (f32 units run in their own launch), block-scaled, against the destination-side
    # block pull of the same f32 weights
    sd32 = {k: v.float() for k, v in sd.items()}
    src32 = DirectWeightSyncSource()
    src32.register(sd32, rank=0, quantize={k: "block" for k in sd32})
    trainer32 = DirectWeightSyncSource()
    handles32 = {k: [h] for k, h in trainer32.register(sd32, rank=0).items()}
    dest = {k: torch.empty(v.shape, dtype=E4M3, device="cuda") for k, v in sd32.items()}
    dest_scales = {k: scale_like("block", v.shape) for k, v in sd32.items()}
    pull32 = DirectWeightSyncDest()
    times = {"src": [], "dst": []}
    for i in range(args.warmup + args.reps):
        ms = refresh_ms(src32, src32._quant_plans)
        asyncio.run(pull32.pull(handles32, dest, block_scales=dest_scales))
        if i >= args.warmup:
            times["src"].append(ms)
            times["dst"].append(pull32.last_pull_ms[0])
    out["block_source_refresh_f32"] = entry(statistics.median(times["src"]), 4 * n, written("block"), copy_gbps)
    out["block_dest_side_pull_f32"] = entry(statistics.median(times["dst"]), 4 * n, written("block"), copy_gbps)
    out["block_source_refresh_f32"]["vs_dest_side_pull"] = round(statistics.median(times["dst"]) / statistics.median(times["src"]), 3)
    bit_exact["full_block_f32"] = exact(src32, {})
    pull32.close()
    asyncio.run(src32.cleanup())
    asyncio.run(trainer32.cleanup())
    out["bit_exact_vs_torch_cuda"] = bit_exact
    print(json.dumps(out))
    assert all(bit_exact.values()), f"source-side quantisation differs from the torch-CUDA rendering: {bit_exact}"


if __name__ == "__main__":
    main()

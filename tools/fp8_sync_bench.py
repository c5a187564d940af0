"""FP8 weight sync on one GPU: the refresh casts of a bf16 or fp32 trainer's staging to float8_e4m3fn
and the N=1 pulls an fp8 generator makes, for the Llama-3-8B state dict (workloads.py shapes).

    python tools/fp8_sync_bench.py [--reps 10] [--warmup 3]

Kernel times come from the plans' own start/done events (tsb_plan_elapsed_ms), medians over warmed,
repeated launches.  Bytes are computed from the shapes (read + written).  Alongside: the card's name
and power limit and its measured device-to-device copy rate (torch copy_ of 4 GiB), which is the
ceiling the traffic rates are compared with.  Prints one JSON line.
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
from torchstore_b200 import _native  # noqa: E402
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource  # noqa: E402

E4M3 = torch.float8_e4m3fn


def copy_rate(reps: int) -> float:
    n = 4 << 30
    a = torch.empty(n, dtype=torch.uint8, device="cuda")
    b = torch.empty_like(a)
    a.random_(0, 255)
    for _ in range(3):
        b.copy_(a)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    rates = []
    for _ in range(5):
        torch.cuda.synchronize()
        e0.record()
        for _ in range(reps):
            b.copy_(a)
        e1.record()
        e1.synchronize()
        rates.append(2 * n * reps / (e0.elapsed_time(e1) / 1e3) / 1e9)
    del a, b
    torch.cuda.empty_cache()
    return statistics.median(rates)


def state_dict(dtype):
    g = torch.Generator(device="cuda").manual_seed(0)
    return {name: torch.randn(shape, device="cuda", generator=g, dtype=torch.float32).to(dtype)
            for name, (shape, _) in workloads.llama_layout().items()}


def numel(sd) -> int:
    return sum(t.numel() for t in sd.values())


def time_refresh(src: DirectWeightSyncSource, warmup: int, reps: int) -> float:
    plans = src._refresh_plans
    times = []
    for i in range(warmup + reps):
        plans.launch()
        plans.synchronize()
        if i >= warmup:
            times.append(plans.elapsed_ms()[0])
    return statistics.median(times)


def time_pull(handles, dest, warmup: int, reps: int) -> tuple[float, dict]:
    sync = DirectWeightSyncDest()
    all_handles = {k: [h] for k, h in handles.items()}
    times = []
    for i in range(warmup + reps):
        asyncio.run(sync.pull(all_handles, dest))
        if i >= warmup:
            times.append(sync.last_pull_ms[0])
    info = sync.plan_info()[0]
    sync.close()
    return statistics.median(times), info


def entry(ms: float, read: int, written: int, copy_gbps: float) -> dict:
    gbps = (read + written) / (ms / 1e3) / 1e9
    return {"kernel_ms": round(ms, 3), "read_GB": round(read / 1e9, 2), "written_GB": round(written / 1e9, 2),
            "GBps": round(gbps, 1), "fraction_of_copy_rate": round(gbps / copy_gbps, 3)}


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

    # (a) bf16 -> e4m3fn refresh, (b) N=1 pull of the fp8 handles, (c) bf16 handles -> e4m3fn destinations
    sd = state_dict(torch.bfloat16)
    n = numel(sd)
    src = DirectWeightSyncSource()
    fp8_handles = src.register(sd, rank=0, transfer_dtype=E4M3)
    vector_rects = _native.plan_info(src._refresh_plans[0]).num_vector_rects
    out["refresh_bf16_to_e4m3"] = entry(time_refresh(src, args.warmup, args.reps), 2 * n, n, copy_gbps)
    out["refresh_bf16_to_e4m3"]["vector_rects"] = vector_rects
    dest = {k: torch.empty(v.shape, dtype=E4M3, device="cuda") for k, v in sd.items()}
    ms, _ = time_pull(fp8_handles, dest, args.warmup, args.reps)
    out["pull_e4m3_handles"] = entry(ms, n, n, copy_gbps)
    assert all(torch.equal(dest[k].view(torch.uint8), src._staging[k][0].view(torch.uint8)) for k in sd)
    asyncio.run(src.cleanup())
    src2 = DirectWeightSyncSource()
    bf16_handles = src2.register(sd, rank=0)
    ms, _ = time_pull(bf16_handles, dest, args.warmup, args.reps)
    out["pull_bf16_handles_into_e4m3"] = entry(ms, 2 * n, n, copy_gbps)
    asyncio.run(src2.cleanup())
    del sd, dest, src, src2, fp8_handles, bf16_handles
    torch.cuda.empty_cache()

    # (a') fp32 master -> e4m3fn refresh
    sd = state_dict(torch.float32)
    src = DirectWeightSyncSource()
    src.register(sd, rank=0, transfer_dtype=E4M3)
    out["refresh_f32_to_e4m3"] = entry(time_refresh(src, args.warmup, args.reps), 4 * n, n, copy_gbps)
    asyncio.run(src.cleanup())
    out["params"] = n
    print(json.dumps(out))


if __name__ == "__main__":
    main()

"""Packed weight sync on one GPU: full-size Llama-3-8B published under its Hugging Face names (q_proj, k_proj,
v_proj, gate_proj, up_proj, ...) and pulled N=1 in bf16 into the vLLM TP1 layout, alternated in the same run:

* ``packed``      -- pull(packed=...) straight into the fused qkv_proj / gate_up_proj;
* ``unfused``     -- the same bytes pulled into HF-named destinations (q, k, v, gate, up kept apart);
* ``unfused_cat`` -- the unfused pull followed by ``torch.cat`` into the fused tensors, what a generator does
  without packed destinations.

    python tools/packed_sync_bench.py [--reps 10] [--warmup 3]

Per variant: the time per sync between CUDA events recorded on the caller's stream around the whole step (the
pull is fenced against that stream on both sides), the copy kernel's own time (last_pull_ms), and the host
overhead per pull (wall-clock time of the pull call minus its kernel time), medians over the repetitions.  The
fused tensors of the packed and the unfused+cat variants are compared bit for bit.  Alongside: the card's name
and power limit, and its device-to-device copy rate (torch copy_ of 4 GiB).  Prints one JSON line.
"""

import argparse
import asyncio
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import workloads  # noqa: E402
from tools.fp8_sync_bench import copy_rate  # noqa: E402
from torchstore_b200 import _native  # noqa: E402
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, NvlinkBuffer, RDMAWeightHandle  # noqa: E402
from torchstore_b200.transport.types import TensorSlice  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    _native.init()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    out = {"gpu": gpu, "copy_GBps_read_plus_write": round(copy_rate(20), 1)}

    hf = workloads.hf_llama_layout(workloads.LLAMA3_8B)
    vl = workloads.vllm_tp_layout(hf, workloads.LLAMA3_8B, 1, 0)
    g = torch.Generator(device="cuda").manual_seed(0)
    handles, sources = {}, {}
    for name, (shape, _) in hf.items():
        t = torch.empty(shape, dtype=torch.bfloat16, device="cuda")
        t.normal_(0, 0.02, generator=g)
        sources[name] = t
        z = (0,) * len(shape)
        handles[name] = [RDMAWeightHandle(NvlinkBuffer(t), TensorSlice(z, (0,), shape, shape, (1,)), 0)]
    packed = {n: parts for n, (_, parts, _) in vl.items() if parts}
    fused = {n: torch.zeros(shape, dtype=torch.bfloat16, device="cuda") for n, (shape, parts, _) in vl.items() if parts}
    plain = {n: torch.zeros(shape, dtype=torch.bfloat16, device="cuda") for n, (shape, parts, _) in vl.items() if not parts}
    # the unfused destinations: one HF-named tensor per part
    split = {p.source: torch.zeros(hf[p.source][0], dtype=torch.bfloat16, device="cuda")
             for parts in packed.values() for p in parts}
    cat_out = {n: torch.zeros_like(t) for n, t in fused.items()}
    dests_packed = {**plain, **fused}
    dests_unfused = {**plain, **split}
    sync_p, sync_u = DirectWeightSyncDest(), DirectWeightSyncDest()

    async def packed_step():
        await sync_p.pull(handles, dests_packed, packed=packed)
        return sync_p.last_pull_ms[0]

    async def unfused_step():
        await sync_u.pull(handles, dests_unfused)
        return sync_u.last_pull_ms[0]

    async def unfused_cat_step():
        ms = await unfused_step()
        for n, parts in packed.items():
            torch.cat([split[p.source] for p in parts], out=cat_out[n])
        return ms

    steps = {"packed": packed_step, "unfused": unfused_step, "unfused_cat": unfused_cat_step}
    res = {k: {"event_ms": [], "kernel_ms": [], "host_ms": []} for k in steps}
    stream = torch.cuda.current_stream()
    order = list(steps)
    for rep in range(args.warmup + args.reps):
        for name in order[rep % 3:] + order[:rep % 3]:  # rotated, so no variant always follows the same one
            step = steps[name]
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            t0 = time.perf_counter()
            kernel = asyncio.run(step())
            wall = (time.perf_counter() - t0) * 1e3
            b.record(stream)
            b.synchronize()
            if rep >= args.warmup:
                res[name]["event_ms"].append(a.elapsed_time(b))
                res[name]["kernel_ms"].append(kernel)
                res[name]["host_ms"].append(wall - kernel)
    nbytes = workloads.state_dict_bytes(hf)
    for name, r in res.items():
        ev = statistics.median(r["event_ms"])
        out[name] = {"ms_per_sync": round(ev, 3), "ms_min": round(min(r["event_ms"]), 3),
                     "ms_max": round(max(r["event_ms"]), 3), "kernel_ms": round(statistics.median(r["kernel_ms"]), 3),
                     "host_overhead_ms": round(statistics.median(r["host_ms"]), 3),
                     "GBps_read_plus_write": round(2 * nbytes / ev / 1e6, 1)}
    out["packed_over_unfused"] = round(out["packed"]["ms_per_sync"] / out["unfused"]["ms_per_sync"], 3)
    out["packed_over_unfused_cat"] = round(out["packed"]["ms_per_sync"] / out["unfused_cat"]["ms_per_sync"], 3)
    out["plan_info_equal"] = sync_p.plan_info() == sync_u.plan_info()
    out["bit_exact"] = all(torch.equal(fused[n].view(torch.int16), cat_out[n].view(torch.int16)) for n in fused) and \
        all(torch.equal(fused[n][p.dest_index], sources[p.source]) for n, parts in packed.items() for p in parts)
    out.update(state_dict_bytes=nbytes, reps=args.reps, warmup=args.warmup)
    sync_p.close()
    sync_u.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

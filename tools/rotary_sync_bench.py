"""Rotary packed weight sync on one GPU: full-size Llama-3-8B published under its torchtitan names (wq, wk, wv, w1,
w3, ..., Meta's interleaved rotary rows in wq and wk) and pulled N=1 in bf16 into the vLLM TP1 layout, alternated in
the same run with the HF-named packed pull of the same bytes:

* ``rotary`` -- pull(packed=vllm_tp_layout(..., source="torchtitan")): every vLLM parameter filled from the torchtitan
  handles, the q and k parts with ``rotary_head_dim=128`` (half-split rows written straight from interleaved ones);
* ``hf``     -- pull(packed=vllm_tp_layout(hf_layout)) from HF-named handles whose q_proj / k_proj are the weights
  permuted by torch (``view / transpose / reshape``), the other names aliasing the same tensors.

    python tools/rotary_sync_bench.py [--reps 10] [--warmup 3]

Per variant: the time per sync between CUDA events around the whole step, the kernels' own time (last_pull_ms) and
the host overhead per pull, medians over the repetitions, the rect count of each compiled plan and whether the two
plans move the same bytes with the same copy/link split.  Every destination of the two variants is compared bit for
bit.  Alongside: the card's name and power limit.  Prints one JSON line.
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
from torchstore_b200 import _native  # noqa: E402
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, NvlinkBuffer, RDMAWeightHandle  # noqa: E402
from torchstore_b200.transport.types import TensorSlice  # noqa: E402

CFG = workloads.LLAMA3_8B


def whole(t):
    z = (0,) * t.dim()
    return [RDMAWeightHandle(NvlinkBuffer(t), TensorSlice(z, (0,), tuple(t.shape), tuple(t.shape), (1,)), 0)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    _native.init()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    out = {"gpu": gpu}

    titan = workloads.llama_layout(CFG)
    hf = workloads.hf_llama_layout(CFG)
    hd = CFG["dim"] // CFG["n_heads"]
    g = torch.Generator(device="cuda").manual_seed(0)
    titan_handles, hf_handles = {}, {}
    for name, (shape, _) in titan.items():
        t = torch.empty(shape, dtype=torch.bfloat16, device="cuda")
        t.normal_(0, 0.02, generator=g)
        titan_handles[name] = whole(t)
        if name.endswith(("attention.wq.weight", "attention.wk.weight")):
            t = t.view(shape[0] // hd, hd // 2, 2, shape[1]).transpose(1, 2).reshape(shape).contiguous()
        hf_handles[workloads.hf_name(name)] = whole(t)
    vt = workloads.vllm_tp_layout(titan, CFG, 1, 0, source="torchtitan")
    vh = workloads.vllm_tp_layout(hf, CFG, 1, 0)
    assert set(vt) == set(vh)
    packed_t = {n: parts for n, (_, parts, _) in vt.items()}
    packed_h = {n: parts for n, (_, parts, _) in vh.items() if parts}
    dests_t = {n: torch.zeros(shape, dtype=torch.bfloat16, device="cuda") for n, (shape, _, _) in vt.items()}
    dests_h = {n: torch.zeros(shape, dtype=torch.bfloat16, device="cuda") for n, (shape, _, _) in vh.items()}
    sync_t, sync_h = DirectWeightSyncDest(), DirectWeightSyncDest()

    async def rotary_step():
        await sync_t.pull(titan_handles, dests_t, packed=packed_t)
        return sync_t.last_pull_ms[0]

    async def hf_step():
        await sync_h.pull(hf_handles, dests_h, packed=packed_h)
        return sync_h.last_pull_ms[0]

    steps = {"rotary": rotary_step, "hf": hf_step}
    res = {k: {"event_ms": [], "kernel_ms": [], "host_ms": []} for k in steps}
    stream = torch.cuda.current_stream()
    order = list(steps)
    for rep in range(args.warmup + args.reps):
        for name in order[rep % 2:] + order[:rep % 2]:  # alternated, so neither always follows the other
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            t0 = time.perf_counter()
            kernel = asyncio.run(steps[name]())
            wall = (time.perf_counter() - t0) * 1e3
            b.record(stream)
            b.synchronize()
            if rep >= args.warmup:
                res[name]["event_ms"].append(a.elapsed_time(b))
                res[name]["kernel_ms"].append(kernel)
                res[name]["host_ms"].append(wall - kernel)
    nbytes = workloads.state_dict_bytes(titan)
    for name, r in res.items():
        ev = statistics.median(r["event_ms"])
        out[name] = {"ms_per_sync": round(ev, 3), "ms_min": round(min(r["event_ms"]), 3),
                     "ms_max": round(max(r["event_ms"]), 3), "kernel_ms": round(statistics.median(r["kernel_ms"]), 3),
                     "host_overhead_ms": round(statistics.median(r["host_ms"]), 3),
                     "GBps_read_plus_write": round(2 * nbytes / ev / 1e6, 1)}
    out["rotary_over_hf"] = round(out["rotary"]["ms_per_sync"] / out["hf"]["ms_per_sync"], 3)
    out["rotary_over_hf_kernel"] = round(out["rotary"]["kernel_ms"] / out["hf"]["kernel_ms"], 3)
    it, ih = sync_t.plan_info()[0], sync_h.plan_info()[0]
    out["rects"] = {"rotary": it["num_rects"], "hf": ih["num_rects"]}
    out["same_bytes_and_split"] = all(it[k] == ih[k] for k in it if "bytes" in k or "link" in k)
    out["bit_exact"] = all(torch.equal(dests_t[n].view(torch.int16), dests_h[n].view(torch.int16)) for n in dests_t)
    out.update(state_dict_bytes=nbytes, reps=args.reps, warmup=args.warmup)
    sync_t.close()
    sync_h.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

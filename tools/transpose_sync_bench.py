"""Transposed packed weight sync on one GPU: Qwen3-30B-A3B's routed experts at full width and expert count (128 x
[2048, 768] per matrix, ``--layers`` layers, 8 by default: 9.66 GB of bf16), published the way a grouped-GEMM trainer
keeps them (input-major ``w1`` / ``w3`` ``[E, dim, ffn]``, ``w2`` ``[E, ffn, dim]``) and pulled N=1 into vLLM's
output-major ``w13_weight [E, 2 ffn, dim]`` / ``w2_weight [E, dim, ffn]``.  Variants, alternated in the same run:

* ``transposed``     -- pull(packed=...) of the grouped handles with ``PackedPart(transpose=True)`` parts;
* ``hf``             -- pull(packed=...) of Hugging Face per-expert handles holding the same values already
  transposed: the copy_rects rate for the same bytes;
* ``pull+torch``     -- pull the grouped tensors into grouped-shaped temporaries, then ``copy_`` their transposes into
  ``w13_weight`` / ``w2_weight`` with torch;
* ``transposed_f32`` -- the transposed pull from float32 grouped handles into the bf16 destinations (fused cast).

    python tools/transpose_sync_bench.py [--layers 8] [--reps 10] [--warmup 3]

Per variant: medians of the time per sync between CUDA events around the whole step, the pull kernels' own time
(last_pull_ms; for pull+torch the pull alone) and the host overhead per sync (wall time minus kernel time), and GB/s of the bytes the sync must read
and write.  Every variant's destinations are compared bit for bit with the transposed pull's.  Alongside: the card's
name and power limit, read in the same call.  Prints one JSON line.
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

CFG = workloads.QWEN3_MOE


def whole(t):
    z = (0,) * t.dim()
    return [RDMAWeightHandle(NvlinkBuffer(t), TensorSlice(z, (0,), tuple(t.shape), tuple(t.shape), (1,)), 0)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=8)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    _native.init()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    out = {"gpu": gpu}

    def experts_only(layout):
        return {k: v for k, v in layout.items() if ".experts." in k or k.endswith("mlp.gate.weight")}

    grouped = experts_only(workloads.qwen3_moe_layout(CFG, n_layers=args.layers, with_embeddings=False,
                                                      grouped_experts=True))
    hf = experts_only(workloads.qwen3_moe_layout(CFG, n_layers=args.layers, with_embeddings=False))
    vt = {k: v for k, v in workloads.vllm_tp_layout(grouped, CFG, 1, 0).items() if v[1]}
    vh = {k: v for k, v in workloads.vllm_tp_layout(hf, CFG, 1, 0).items() if v[1]}
    assert set(vt) == set(vh)
    g = torch.Generator(device="cuda").manual_seed(0)
    g_handles, f_handles, h_handles, temps = {}, {}, {}, {}
    for name, (shape, _) in grouped.items():
        if ".experts.w" not in name:
            continue
        t = torch.empty(shape, dtype=torch.bfloat16, device="cuda")
        t.normal_(0, 0.02, generator=g)
        g_handles[name] = whole(t)
        f_handles[name] = whole(t.float())
        temps[name] = torch.empty_like(t)
        base, w = name.rsplit(".", 1)
        hname = {"w1": "gate_proj", "w3": "up_proj", "w2": "down_proj"}[w]
        for e in range(shape[0]):  # the HF per-expert tensor: the same values, output-major
            h_handles[f"{base}.{e}.{hname}.weight"] = whole(t[e].t().contiguous())
    packed_t = {n: parts for n, (_, parts, _) in vt.items()}
    packed_h = {n: parts for n, (_, parts, _) in vh.items()}
    dests_t = {n: torch.zeros(shape, dtype=torch.bfloat16, device="cuda") for n, (shape, _, _) in vt.items()}
    dests_o = {n: torch.zeros(shape, dtype=torch.bfloat16, device="cuda") for n, (shape, _, _) in vt.items()}
    syncs = {k: DirectWeightSyncDest() for k in ("transposed", "hf", "pull+torch", "transposed_f32")}

    async def transposed():
        await syncs["transposed"].pull(g_handles, dests_t, packed=packed_t)
        return syncs["transposed"].last_pull_ms[0]

    async def hf_step():
        await syncs["hf"].pull(h_handles, dests_o, packed=packed_h)
        return syncs["hf"].last_pull_ms[0]

    async def pull_torch():
        await syncs["pull+torch"].pull(g_handles, temps)
        for i in range(args.layers):
            ex = f"model.layers.{i}.mlp.experts."
            f = CFG["moe_ffn"]
            w13 = dests_o[ex + "w13_weight"]
            w13[:, :f].copy_(temps[ex + "w1"].transpose(-2, -1))
            w13[:, f:].copy_(temps[ex + "w3"].transpose(-2, -1))
            dests_o[ex + "w2_weight"].copy_(temps[ex + "w2"].transpose(-2, -1))
        return syncs["pull+torch"].last_pull_ms[0]

    async def transposed_f32():
        await syncs["transposed_f32"].pull(f_handles, dests_o, packed=packed_t)
        return syncs["transposed_f32"].last_pull_ms[0]

    steps = {"transposed": transposed, "hf": hf_step, "pull+torch": pull_torch, "transposed_f32": transposed_f32}
    res = {k: {"event_ms": [], "kernel_ms": [], "host_ms": []} for k in steps}
    stream = torch.cuda.current_stream()
    order = list(steps)
    for rep in range(args.warmup + args.reps):
        for name in order[rep % len(order):] + order[:rep % len(order)]:  # rotated: no variant always follows another
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            t0 = time.perf_counter()
            kernel = asyncio.run(steps[name]())
            b.record(stream)
            b.synchronize()
            wall = (time.perf_counter() - t0) * 1e3
            if rep >= args.warmup:
                res[name]["event_ms"].append(a.elapsed_time(b))
                res[name]["kernel_ms"].append(kernel)
                res[name]["host_ms"].append(wall - kernel)
    nbytes = sum(t.numel() * t.element_size() for t in temps.values())
    moved = {"transposed": 2 * nbytes, "hf": 2 * nbytes, "pull+torch": 2 * nbytes, "transposed_f32": 3 * nbytes}
    for name, r in res.items():
        ev = statistics.median(r["event_ms"])
        out[name] = {"ms_per_sync": round(ev, 3), "ms_min": round(min(r["event_ms"]), 3),
                     "ms_max": round(max(r["event_ms"]), 3), "kernel_ms": round(statistics.median(r["kernel_ms"]), 3),
                     "host_overhead_ms": round(statistics.median(r["host_ms"]), 3),
                     "GBps_read_plus_write": round(moved[name] / ev / 1e6, 1)}
    out["transposed_over_pull_torch"] = round(out["transposed"]["ms_per_sync"] / out["pull+torch"]["ms_per_sync"], 3)
    out["transposed_over_hf_kernel"] = round(out["transposed"]["kernel_ms"] / out["hf"]["kernel_ms"], 3)
    out["transposed_f32_over_hf_kernel"] = round(out["transposed_f32"]["kernel_ms"] / out["hf"]["kernel_ms"], 3)
    exact = {}
    for name in ("hf", "pull+torch", "transposed_f32"):  # they share dests_o: run each once more, then compare
        for t in dests_o.values():
            t.fill_(0)
        asyncio.run(steps[name]())
        torch.cuda.synchronize()
        exact[name] = all(torch.equal(dests_t[n].view(torch.int16), dests_o[n].view(torch.int16)) for n in dests_t)
    out["bit_exact_vs_transposed"] = exact
    out["transpose_tiles"] = _native.plan_info(next(iter(syncs["transposed"]._transpose_plans.values()))).num_tiles
    out.update(expert_bytes_bf16=nbytes, layers=args.layers, reps=args.reps, warmup=args.warmup)
    for s in syncs.values():
        s.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()

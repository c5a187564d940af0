"""Dequantising weight sync on one GPU: the Llama-3-8B linear weights (wq wk wv wo w1 w2 w3), quantised on
the GPU by the existing block-, channel- and tensor-scaled pulls, published as scaled fp8 handles and
pulled back N=1 into bf16 for each granularity, alternated in the same run with the unscaled fused
e4m3fn -> bf16 pull of the same fp8 bytes.

    python tools/dequant_fp8_sync_bench.py [--reps 10] [--warmup 3]

Kernel times come from the plans' own start/done events (last_pull_ms), medians over warmed, repeated
launches.  Bytes are computed from the shapes: each pull reads the fp8 weights (plus the scales) once and
writes bf16.  Alongside: the card's name and power limit and its measured device-to-device copy rate
(torch copy_ of 4 GiB), the ceiling the rates are compared with.  The last pull of each granularity is
checked bit for bit against the torch-CUDA rendering (q.float() * s).to(bf16).  Prints one JSON line.
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
from oracle.dequant_fp8_oracle import torch_dequantize  # noqa: E402
from tools.fp8_sync_bench import copy_rate, entry  # noqa: E402
from torchstore_b200 import _native  # noqa: E402
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource  # noqa: E402

E4M3 = torch.float8_e4m3fn
LINEAR = {"wq", "wk", "wv", "wo", "w1", "w2", "w3"}
KW = {"block": "block_scales", "channel": "channel_scales", "tensor": "tensor_scales"}


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
    trainer = DirectWeightSyncSource()
    bf16_handles = {k: [h] for k, h in trainer.register(sd, rank=0).items()}

    # quantise on the GPU with the existing pulls: one fp8 copy and its scales per granularity
    fp8, scales = {}, {}
    for gran in KW:
        fp8[gran] = {k: torch.empty(v.shape, dtype=E4M3, device="cuda") for k, v in sd.items()}
        if gran == "block":
            scales[gran] = {k: torch.empty(-(-v.shape[0] // 128), -(-v.shape[1] // 128), device="cuda") for k, v in sd.items()}
        elif gran == "channel":
            scales[gran] = {k: torch.empty(v.shape[0], 1, device="cuda") for k, v in sd.items()}
        else:
            scales[gran] = {k: torch.empty((), device="cuda") for k in sd}
        q = DirectWeightSyncDest()
        asyncio.run(q.pull(bf16_handles, fp8[gran], **{KW[gran]: scales[gran]}))
        q.close()
    del bf16_handles
    asyncio.run(trainer.cleanup())
    del sd

    n = sum(v.numel() for v in fp8["block"].values())
    generators, forms = [], {}
    for gran in KW:
        gen = DirectWeightSyncSource()
        h = {k: [v] for k, v in gen.register(fp8[gran], rank=0, **{KW[gran]: scales[gran]}).items()}
        generators.append(gen)
        forms[f"{gran}_dequant_pull"] = (DirectWeightSyncDest(), h, gran)
    gen = DirectWeightSyncSource()
    generators.append(gen)
    forms["unscaled_e4m3_to_bf16_pull"] = (DirectWeightSyncDest(), {k: [v] for k, v in gen.register(fp8["block"], rank=0).items()},
                                           None)
    dest = {k: torch.empty(v.shape, dtype=torch.bfloat16, device="cuda") for k, v in fp8["block"].items()}
    times = {k: [] for k in forms}
    for i in range(args.warmup + args.reps):  # alternate the four pulls
        for key, (sync, h, _) in forms.items():
            asyncio.run(sync.pull(h, dest))
            if i >= args.warmup:
                times[key].append(sync.last_pull_ms[0])
    med = {k: statistics.median(v) for k, v in times.items()}
    for key, (sync, _, gran) in forms.items():
        n_s = sum(s.numel() for s in scales[gran].values()) if gran else 0
        out[key] = entry(med[key], n + 4 * n_s, 2 * n, copy_gbps)
        plans = sync._dequant_plans if gran else sync._native_plans
        out[key].update(ctas=plans.info()[0]["grid"])
    unscaled = med["unscaled_e4m3_to_bf16_pull"]
    for gran in KW:
        out[f"{gran}_dequant_pull"]["vs_unscaled"] = round(unscaled / med[f"{gran}_dequant_pull"], 3)

    exact = {}
    for gran in KW:
        sync, h, _ = forms[f"{gran}_dequant_pull"]
        asyncio.run(sync.pull(h, dest))
        torch.cuda.synchronize()
        ok = True
        for k in names:
            want = torch_dequantize(fp8[gran][k], scales[gran][k], gran)
            ok &= torch.equal(dest[k].view(torch.int16), want.view(torch.int16))
            del want
        exact[gran] = bool(ok)
    out["bit_exact_vs_torch_cuda"] = exact
    out["params"] = n
    for sync, _, _ in forms.values():
        sync.close()
    for gen in generators:
        asyncio.run(gen.cleanup())
    print(json.dumps(out))
    assert all(exact.values()), f"dequantising pull differs from the torch-CUDA rendering: {exact}"


if __name__ == "__main__":
    main()

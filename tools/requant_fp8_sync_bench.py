"""Requantising weight sync on one GPU: the Llama-3-8B linear weights (wq wk wv wo w1 w2 w3), quantised on the
GPU by the existing block-scaled pull, published as block-scaled fp8 handles and pulled N=1 with
requantize=True into block-, channel- and tensor-scaled fp8 destinations, alternated in the same run with
the two-step route users take without it: a dequantising pull into an f32 temporary, then a quantising pull
from it into block-scaled fp8.

    python tools/requant_fp8_sync_bench.py [--reps 10] [--warmup 3]

Kernel times come from the plans' own start/done events (last_pull_ms), medians over warmed, repeated
launches.  Bytes are computed from the shapes: a requantising pull reads the fp8 weights once (twice into
per-tensor destinations, whose pass 1 only folds the amax) plus the source scales and writes the fp8 bytes
and the destination scales; the two-step route reads 1 + 4 and writes 4 + 1 bytes per element.  Alongside:
the card's name and power limit and its measured device-to-device copy rate (torch copy_ of 4 GiB), the
ceiling the rates are compared with.  The last pull of each destination granularity is checked bit for bit
against the torch-CUDA composition (torch_dequantize to f32, then torch_quantize), and the two-step route's
output against the fused block pull.  Prints one JSON line.
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
from oracle.requant_fp8_oracle import torch_requantize  # noqa: E402
from tools.fp8_sync_bench import copy_rate, entry  # noqa: E402
from torchstore_b200 import _native  # noqa: E402
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource  # noqa: E402

E4M3 = torch.float8_e4m3fn
LINEAR = {"wq", "wk", "wv", "wo", "w1", "w2", "w3"}
KW = {"block": "block_scales", "channel": "channel_scales", "tensor": "tensor_scales"}


def scale_like(gran: str, shape) -> torch.Tensor:
    if gran == "block":
        return torch.empty(-(-shape[0] // 128), -(-shape[1] // 128), device="cuda")
    if gran == "channel":
        return torch.empty(shape[0], 1, device="cuda")
    return torch.empty((), device="cuda")


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
    # the block-scaled checkpoint, quantised on the GPU by the existing pull
    fp8 = {k: torch.empty(v.shape, dtype=E4M3, device="cuda") for k, v in sd.items()}
    src_scales = {k: scale_like("block", v.shape) for k, v in sd.items()}
    q = DirectWeightSyncDest()
    asyncio.run(q.pull(bf16_handles, fp8, block_scales=src_scales))
    q.close()
    del bf16_handles
    asyncio.run(trainer.cleanup())
    del sd

    n = sum(v.numel() for v in fp8.values())
    n_src_scales = sum(s.numel() for s in src_scales.values())
    gen = DirectWeightSyncSource()
    handles = {k: [v] for k, v in gen.register(fp8, rank=0, block_scales=src_scales).items()}
    dest = {k: torch.empty(v.shape, dtype=E4M3, device="cuda") for k, v in fp8.items()}
    dest_scales = {gran: {k: scale_like(gran, v.shape) for k, v in fp8.items()} for gran in KW}
    forms = {f"block_to_{gran}_requant_pull": (DirectWeightSyncDest(), gran) for gran in KW}
    # the two-step route: dequantise into an f32 temporary, then quantise from it
    tmp = {k: torch.empty(v.shape, device="cuda") for k, v in fp8.items()}
    tmp_src = DirectWeightSyncSource()
    tmp_handles = {k: [v] for k, v in tmp_src.register(tmp, rank=0).items()}
    two_dq, two_q = DirectWeightSyncDest(), DirectWeightSyncDest()
    two_dest = {k: torch.empty(v.shape, dtype=E4M3, device="cuda") for k, v in fp8.items()}
    two_scales = {k: scale_like("block", v.shape) for k, v in fp8.items()}

    times = {k: [] for k in list(forms) + ["two_step_f32_route_to_block"]}
    for i in range(args.warmup + args.reps):  # alternate the four routes
        for key, (sync, gran) in forms.items():
            asyncio.run(sync.pull(handles, dest, **{KW[gran]: dest_scales[gran]}, requantize=True))
            if i >= args.warmup:
                times[key].append(sync.last_pull_ms[0])
        asyncio.run(two_dq.pull(handles, tmp))
        asyncio.run(two_q.pull(tmp_handles, two_dest, block_scales=two_scales))
        if i >= args.warmup:
            times["two_step_f32_route_to_block"].append(two_dq.last_pull_ms[0] + two_q.last_pull_ms[0])
    med = {k: statistics.median(v) for k, v in times.items()}
    for key, (sync, gran) in forms.items():
        n_dst_scales = sum(s.numel() for s in dest_scales[gran].values())
        read = (2 if gran == "tensor" else 1) * n + 4 * n_src_scales
        out[key] = entry(med[key], read, n + 4 * n_dst_scales, copy_gbps)
        out[key].update(ctas=sync._requant_plans.info()[0]["grid"])
    key = "two_step_f32_route_to_block"
    out[key] = entry(med[key], 5 * n + 4 * n_src_scales, 5 * n + 4 * sum(s.numel() for s in two_scales.values()), copy_gbps)
    out["block_to_block_requant_pull"]["vs_two_step"] = round(med[key] / med["block_to_block_requant_pull"], 3)

    exact = {}
    for key, (sync, gran) in forms.items():
        asyncio.run(sync.pull(handles, dest, **{KW[gran]: dest_scales[gran]}, requantize=True))
        torch.cuda.synchronize()
        ok = True
        for k in names:
            want_q, want_s = torch_requantize(fp8[k], src_scales[k], "block", 0, 0, gran)
            ok &= torch.equal(dest[k].view(torch.uint8), want_q.view(torch.uint8))
            ok &= torch.equal(dest_scales[gran][k].view(torch.int32), want_s.reshape(dest_scales[gran][k].shape).view(torch.int32))
            if gran == "block":
                ok &= torch.equal(two_dest[k].view(torch.uint8), dest[k].view(torch.uint8))
                ok &= torch.equal(two_scales[k].view(torch.int32), dest_scales[gran][k].view(torch.int32))
            del want_q, want_s
        exact[gran] = bool(ok)
    out["bit_exact_vs_torch_cuda"] = exact
    out["params"] = n
    for sync, _ in forms.values():
        sync.close()
    two_dq.close()
    two_q.close()
    asyncio.run(gen.cleanup())
    asyncio.run(tmp_src.cleanup())
    print(json.dumps(out))
    assert all(exact.values()), f"requantising pull differs from the torch-CUDA composition: {exact}"


if __name__ == "__main__":
    main()

"""Verbatim weight sync on one GPU: the Llama-3-8B linear weights (wq wk wv wo w1 w2 w3) quantised on the source
by register(quantize=g) into block-, channel- and tensor-scaled fp8 staging, then pulled N=1 into fp8
destinations of the same granularity with verbatim=True (the fp8 bytes and scale rectangles in one copy plan),
alternated in the same run with requantize=True into the same destinations and with the raw fp8 byte pull
(no scale dicts), which moves the same bytes without the scale rectangles.

    python tools/verbatim_fp8_sync_bench.py [--reps 10] [--warmup 3]

Kernel times come from the plans' own start/done events (last_pull_ms), medians over warmed, repeated
launches.  Bytes are computed from the shapes: a verbatim pull reads and writes 1 byte per element plus the
scales (4 bytes each); a requantising pull reads the fp8 weights once (twice into per-tensor destinations, whose
pass 1 only folds the amax) plus the source scales and writes the fp8 bytes and the destination scales.
Alongside: the card's name and power limit and its measured device-to-device copy rate (torch copy_ of 4 GiB),
the ceiling the rates are compared with.  The last verbatim pull of each granularity is checked bit for bit
against the source's staging bytes and scales.  Prints one JSON line.
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
    n = sum(v.numel() for v in sd.values())
    dest = {k: torch.empty(v.shape, dtype=E4M3, device="cuda") for k, v in sd.items()}
    exact = {}
    for gran in KW:
        trainer = DirectWeightSyncSource()
        handles = {k: [h] for k, h in trainer.register(sd, rank=0, quantize={k: gran for k in names}).items()}
        scales = {k: scale_like(gran, v.shape) for k, v in sd.items()}
        n_scales = sum(s.numel() for s in scales.values())
        syncs = {"verbatim": DirectWeightSyncDest(), "requant": DirectWeightSyncDest(), "raw": DirectWeightSyncDest()}
        kw = {"verbatim": {KW[gran]: scales, "verbatim": True}, "requant": {KW[gran]: scales, "requantize": True},
              "raw": {}}
        times = {k: [] for k in syncs}
        for i in range(args.warmup + args.reps):  # alternate the three routes
            for route, sync in syncs.items():
                asyncio.run(sync.pull(handles, dest, **kw[route]))
                if i >= args.warmup:
                    times[route].append(sync.last_pull_ms[0])
        med = {k: statistics.median(v) for k, v in times.items()}
        assert not any(syncs["verbatim"]._fp8_plans), "a verbatim pull built an fp8 plan"
        key = f"{gran}_verbatim_pull"
        out[key] = entry(med["verbatim"], n + 4 * n_scales, n + 4 * n_scales, copy_gbps)
        out[key]["vs_requantize"] = round(med["requant"] / med["verbatim"], 3)
        out[key]["vs_raw_bytes"] = round(med["raw"] / med["verbatim"], 3)
        out[key]["plan"] = syncs["verbatim"].plan_info()[0]
        read = (2 if gran == "tensor" else 1) * n + 4 * n_scales
        out[f"{gran}_requantize_pull"] = entry(med["requant"], read, n + 4 * n_scales, copy_gbps)
        out[f"{gran}_raw_byte_pull"] = entry(med["raw"], n, n, copy_gbps)
        asyncio.run(syncs["verbatim"].pull(handles, dest, **{KW[gran]: scales}, verbatim=True))
        torch.cuda.synchronize()
        ok = True
        for k in names:
            q, s, _ = trainer._quantized[k]
            ok &= torch.equal(dest[k].view(torch.uint8), q.view(torch.uint8))
            ok &= torch.equal(scales[k].reshape(-1).view(torch.int32), s.reshape(-1).view(torch.int32))
        exact[gran] = bool(ok)
        for sync in syncs.values():
            sync.close()
        asyncio.run(trainer.cleanup())
    out["bit_exact_vs_source_staging"] = exact
    out["params"] = n
    print(json.dumps(out))
    assert all(exact.values()), f"verbatim pull differs from the source staging: {exact}"


if __name__ == "__main__":
    main()

"""Scaled INT8 weight sync on one GPU: the N=1 pull of the Llama-3-8B bf16 state dict's linear weights (wq wk wv
wo w1 w2 w3) into int8 with float32 scales per 128x128 block, per row and per matrix, each alternated in the same
run with the float8_e4m3fn pull of the same granularity.  The two pulls of a granularity move the same bytes (the
same source reads, 1 byte written per element, the same scales); only the narrowing and the scale step differ.

    python tools/int8_sync_bench.py [--reps 10] [--warmup 3]

Kernel times come from the plans' own start/done events (last_pull_ms), medians over warmed, repeated launches.
Alongside: the card's name and power limit and its measured device-to-device copy rate (torch copy_ of 4 GiB).
The last int8 pull of each granularity is checked bit for bit against the torch-CUDA rendering of the formula
(int8_oracle.torch_quantize), at full size.  Prints one JSON line.
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
from oracle.int8_oracle import scale_shape, torch_quantize  # noqa: E402
from tools.fp8_sync_bench import copy_rate, entry  # noqa: E402
from torchstore_b200 import _native  # noqa: E402
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource  # noqa: E402

LINEAR = {"wq", "wk", "wv", "wo", "w1", "w2", "w3"}
GRANULARITIES = ("block", "channel", "tensor")


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
    sd = {k: torch.randn(layout[k][0], device="cuda", generator=g, dtype=torch.float32).to(torch.bfloat16) for k in names}
    src = DirectWeightSyncSource()
    handles = {k: [h] for k, h in src.register(sd, rank=0).items()}
    n = sum(v.numel() for v in sd.values())

    forms = {}
    for gran in GRANULARITIES:
        scales = {k: torch.empty(scale_shape(gran, tuple(v.shape)), device="cuda") for k, v in sd.items()}
        for fmt, dtype in (("int8", torch.int8), ("fp8", torch.float8_e4m3fn)):
            q = {k: torch.empty(v.shape, dtype=dtype, device="cuda") for k, v in sd.items()}
            forms[f"{gran}_{fmt}_pull"] = (DirectWeightSyncDest(), q, {f"{gran}_scales": scales})
    times = {k: [] for k in forms}
    for i in range(args.warmup + args.reps):  # alternate every pull
        for key, (sync, q, kw) in forms.items():
            asyncio.run(sync.pull(handles, q, **kw))
            if i >= args.warmup:
                times[key].append(sync.last_pull_ms[0])
    for key, (sync, q, kw) in forms.items():
        n_s = sum(s.numel() for s in next(iter(kw.values())).values())
        reads = 4 * n if key.startswith("tensor") else 2 * n  # the per-tensor pull reads the source twice
        out[key] = entry(statistics.median(times[key]), reads, n + 4 * n_s, copy_gbps)
    for gran in GRANULARITIES:
        i8, f8 = out[f"{gran}_int8_pull"]["kernel_ms"], out[f"{gran}_fp8_pull"]["kernel_ms"]
        out[f"{gran}_int8_over_fp8"] = round(i8 / f8, 4)

    exact = {}
    for gran in GRANULARITIES:
        sync, q, kw = forms[f"{gran}_int8_pull"]
        scales = kw[f"{gran}_scales"]
        asyncio.run(sync.pull(handles, q, **kw))
        torch.cuda.synchronize()
        ok = True
        for k in names:
            want_q, want_s = torch_quantize(sd[k], gran)
            ok &= torch.equal(q[k], want_q) and torch.equal(scales[k].view(torch.int32), want_s.view(torch.int32))
            del want_q, want_s
        exact[gran] = bool(ok)
    out["bit_exact_vs_torch_cuda"] = exact
    out["params"] = n
    for sync, _, _ in forms.values():
        sync.close()
    asyncio.run(src.cleanup())
    print(json.dumps(out))
    assert all(exact.values()), f"int8 pull differs from the torch-CUDA rendering: {exact}"


if __name__ == "__main__":
    main()

"""Block-scaled FP8 weight sync on one GPU: the N=1 pull of the Llama-3-8B bf16 state dict's linear
weights (wq wk wv wo w1 w2 w3) into float8_e4m3fn with one float32 scale_inv per 128x128 block, next to
the plain fused bf16 -> e4m3fn pull of the same parameters (alternated in the same run).

    python tools/block_fp8_sync_bench.py [--reps 10] [--warmup 3]

Kernel times come from the plans' own start/done events (last_pull_ms), medians over warmed, repeated
launches.  Bytes are computed from the shapes (bf16 read + fp8 and scales written).  Alongside: the
card's name and power limit and its measured device-to-device copy rate (torch copy_ of 4 GiB), the
ceiling the rates are compared with.  The last block-scaled pull is checked bit for bit against the
torch-CUDA rendering of the formula.  Prints one JSON line.
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
from oracle.block_fp8_oracle import torch_quantize  # noqa: E402
from tools.fp8_sync_bench import copy_rate, entry  # noqa: E402
from torchstore_b200 import _native  # noqa: E402
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource  # noqa: E402

E4M3 = torch.float8_e4m3fn
LINEAR = {"wq", "wk", "wv", "wo", "w1", "w2", "w3"}


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
    q = {k: torch.empty(v.shape, dtype=E4M3, device="cuda") for k, v in sd.items()}
    scales = {k: torch.empty(-(-v.shape[0] // 128), -(-v.shape[1] // 128), device="cuda") for k, v in sd.items()}
    n = sum(v.numel() for v in sd.values())
    n_scales = sum(s.numel() for s in scales.values())

    block, plain = DirectWeightSyncDest(), DirectWeightSyncDest()
    tb, tp = [], []
    for i in range(args.warmup + args.reps):  # alternate the two pulls
        asyncio.run(block.pull(handles, q, block_scales=scales))
        if i >= args.warmup:
            tb.append(block.last_pull_ms[0])
        asyncio.run(plain.pull(handles, q))
        if i >= args.warmup:
            tp.append(plain.last_pull_ms[0])
    info = block._block_plans.info()[0]
    out["block_fp8_pull"] = entry(statistics.median(tb), 2 * n, n + 4 * n_scales, copy_gbps)
    out["block_fp8_pull"].update(blocks=info["num_tiles"], scale_bytes=4 * n_scales)
    out["plain_e4m3_pull"] = entry(statistics.median(tp), 2 * n, n, copy_gbps)

    asyncio.run(block.pull(handles, q, block_scales=scales))
    torch.cuda.synchronize()
    exact = True
    for k in names:
        want_q, want_s = torch_quantize(sd[k])
        exact &= torch.equal(q[k].view(torch.uint8), want_q.view(torch.uint8)) and \
            torch.equal(scales[k].view(torch.int32), want_s.view(torch.int32))
        del want_q, want_s
    out["bit_exact_vs_torch_cuda"] = bool(exact)
    out["params"] = n
    block.close()
    plain.close()
    asyncio.run(src.cleanup())
    print(json.dumps(out))
    assert exact, "block-scaled pull differs from the torch-CUDA rendering"


if __name__ == "__main__":
    main()

"""Power-of-two (UE8M0) scales on one GPU: every quantising route of the Llama-3-8B linear weights (wq wk wv wo w1 w2
w3, bf16, N=1) run with ``scale_fmt=None`` and ``scale_fmt="ue8m0"`` alternated in the same run:

* the block-, channel- and tensor-scaled pulls from local bf16 handles;
* the block -> block requantising pull from block-scaled fp8 handles;
* the block- and channel-scaled source refresh (``register(quantize=...)``).

    python tools/ue8m0_bench.py [--reps 10] [--warmup 3]

Kernel times come from the plans' own start/done events, medians over warmed, repeated launches.  Alongside: the
card's name and power limit and its measured device-to-device copy rate (torch copy_ of 4 GiB).  Every route's result,
in both formats, is checked bit for bit at full size against the torch-CUDA rendering of its formula
(ue8m0_oracle.torch_quantize / torch_requantize).  Prints one JSON line.
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
from oracle.ue8m0_oracle import torch_quantize, torch_requantize  # noqa: E402
from tools.fp8_sync_bench import copy_rate, entry  # noqa: E402
from tools.source_quant_bench import KW, LINEAR, scale_like  # noqa: E402
from torchstore_b200 import _native  # noqa: E402
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource  # noqa: E402

E4M3 = torch.float8_e4m3fn
FORMATS = (None, "ue8m0")


def same(q: torch.Tensor, s: torch.Tensor, want: tuple) -> bool:
    return bool(torch.equal(q.view(torch.uint8), want[0].view(torch.uint8)) and
                torch.equal(s.view(torch.int32), want[1].reshape(s.shape).view(torch.int32)))


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
    out["params"] = n

    trainer = DirectWeightSyncSource()
    handles = {k: [h] for k, h in trainer.register(sd, rank=0).items()}
    # block-scaled fp8 handles (float32 scales) for the requantising route
    fp8_sd, fp8_scales = {}, {}
    for k, v in sd.items():
        fp8_sd[k], fp8_scales[k] = torch_quantize(v, "block")
    fp8_src = DirectWeightSyncSource()
    fp8_handles = {k: [h] for k, h in fp8_src.register(fp8_sd, rank=0, block_scales=fp8_scales).items()}
    # one fp8 destination dict for every pull (each route and format has its own plan over it); a route's result
    # is checked right after its last run
    dest = {k: torch.empty(v.shape, dtype=E4M3, device="cuda") for k, v in sd.items()}
    routes = {}  # (route, fmt) -> (run() -> kernel ms, check() -> bit-exact)

    def check_pull(scales, want):
        return all(same(dest[k], scales[k], want(k)) for k in sd)

    for fmt in FORMATS:
        for gran in ("block", "channel", "tensor"):
            scales = {k: scale_like(gran, v.shape) for k, v in sd.items()}
            sync = DirectWeightSyncDest()

            def run(sync=sync, scales=scales, gran=gran, fmt=fmt):
                asyncio.run(sync.pull(handles, dest, **{KW[gran]: scales}, scale_fmt=fmt))
                return sync.last_pull_ms[0]

            routes[(f"{gran}_pull", fmt)] = (run, lambda scales=scales, gran=gran, fmt=fmt: check_pull(
                scales, lambda k: torch_quantize(sd[k], gran, scale_fmt=fmt)))
        scales = {k: scale_like("block", v.shape) for k, v in sd.items()}
        sync = DirectWeightSyncDest()

        def run(sync=sync, scales=scales, fmt=fmt):
            asyncio.run(sync.pull(fp8_handles, dest, block_scales=scales, requantize=True, scale_fmt=fmt))
            return sync.last_pull_ms[0]

        routes[("block_to_block_requant_pull", fmt)] = (run, lambda scales=scales, fmt=fmt: check_pull(
            scales, lambda k: torch_requantize(fp8_sd[k], fp8_scales[k], "block", 0, 0, "block", scale_fmt=fmt)))
        for gran in ("block", "channel"):
            src = DirectWeightSyncSource()
            src.register(sd, rank=0, quantize={k: gran for k in sd}, scale_fmt=fmt)

            def run(src=src):
                src.refresh()
                return src._quant_plans.elapsed_ms()[0]

            def check(src=src, gran=gran, fmt=fmt):
                return all(same(q, s, torch_quantize(sd[k], gran, scale_fmt=fmt)) for k, (q, s, _) in src._quantized.items())

            routes[(f"{gran}_source_refresh", fmt)] = (run, check)

    order = list(dict.fromkeys(r for r, _ in routes))
    times = {key: [] for key in routes}
    bit_exact = {}
    for i in range(args.warmup + args.reps):  # alternate every route and format
        for r in order:
            for fmt in FORMATS:
                run, check = routes[(r, fmt)]
                ms = run()
                if i >= args.warmup:
                    times[(r, fmt)].append(ms)
                if i == args.warmup + args.reps - 1:
                    bit_exact[f"{r}_{fmt or 'float32'}"] = check()
    for r in order:
        read = {"tensor_pull": 4 * n, "block_to_block_requant_pull": n}.get(r, 2 * n)
        gran = "block" if r.startswith("block") else "channel" if r.startswith("channel") else "tensor"
        written = n + 4 * sum(scale_like(gran, v.shape).numel() for v in sd.values())
        f32, ue = statistics.median(times[(r, None)]), statistics.median(times[(r, "ue8m0")])
        out[r] = {"float32": entry(f32, read, written, copy_gbps), "ue8m0": entry(ue, read, written, copy_gbps),
                  "ue8m0_vs_float32": round(ue / f32, 3),
                  "spread_ms": {fmt or "float32": [round(min(times[(r, fmt)]), 4), round(max(times[(r, fmt)]), 4)]
                                for fmt in FORMATS}}
    out["bit_exact_vs_torch_cuda"] = bit_exact
    print(json.dumps(out))
    assert all(bit_exact.values()), f"a route differs from the torch-CUDA rendering: {bit_exact}"


if __name__ == "__main__":
    main()

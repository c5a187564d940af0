"""Per-channel and per-tensor scaled FP8 weight sync on one GPU: the N=1 pull of the Llama-3-8B bf16 state
dict's linear weights (wq wk wv wo w1 w2 w3) into float8_e4m3fn with one float32 scale per row
(channel_scales) and per matrix (tensor_scales), next to the 128x128 block-scaled pull and the plain fused
bf16 -> e4m3fn pull of the same parameters (all four alternated in the same run).

    python tools/scaled_fp8_sync_bench.py [--reps 10] [--warmup 3]

Kernel times come from the plans' own start/done events (last_pull_ms), medians over warmed, repeated
launches.  Bytes are computed from the shapes: the per-channel pull reads the bf16 source once, the
per-tensor pull twice (amax pass, then quantise pass); both write fp8 and scales.  Alongside: the card's
name and power limit and its measured device-to-device copy rate (torch copy_ of 4 GiB), the ceiling the
rates are compared with.  The last pull of each of the two new forms is checked bit for bit against the
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
from oracle.scaled_fp8_oracle import torch_quantize  # noqa: E402
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

    def fp8_like():
        return {k: torch.empty(v.shape, dtype=E4M3, device="cuda") for k, v in sd.items()}

    qc, qt, qb = fp8_like(), fp8_like(), fp8_like()
    cs = {k: torch.empty(v.shape[0], 1, device="cuda") for k, v in sd.items()}
    tsc = {k: torch.empty((), device="cuda") for k in sd}
    bs = {k: torch.empty(-(-v.shape[0] // 128), -(-v.shape[1] // 128), device="cuda") for k, v in sd.items()}
    n = sum(v.numel() for v in sd.values())
    n_cs, n_ts, n_bs = (sum(s.numel() for s in d.values()) for d in (cs, tsc, bs))

    forms = {
        "channel_fp8_pull": (DirectWeightSyncDest(), qc, {"channel_scales": cs}),
        "tensor_fp8_pull": (DirectWeightSyncDest(), qt, {"tensor_scales": tsc}),
        "block_fp8_pull": (DirectWeightSyncDest(), qb, {"block_scales": bs}),
        "plain_e4m3_pull": (DirectWeightSyncDest(), qb, {}),
    }
    times = {k: [] for k in forms}
    for i in range(args.warmup + args.reps):  # alternate the four pulls
        for key, (sync, q, kw) in forms.items():
            asyncio.run(sync.pull(handles, q, **kw))
            if i >= args.warmup:
                times[key].append(sync.last_pull_ms[0])
    med = {k: statistics.median(v) for k, v in times.items()}
    out["channel_fp8_pull"] = entry(med["channel_fp8_pull"], 2 * n, n + 4 * n_cs, copy_gbps)
    out["channel_fp8_pull"].update(scales=n_cs, ctas=forms["channel_fp8_pull"][0]._scaled_plans.info()[0]["num_tiles"])
    out["tensor_fp8_pull"] = entry(med["tensor_fp8_pull"], 4 * n, n + 4 * n_ts, copy_gbps)
    out["tensor_fp8_pull"].update(scales=n_ts, ctas_per_pass=forms["tensor_fp8_pull"][0]._scaled_plans.info()[0]["num_tiles"])
    out["block_fp8_pull"] = entry(med["block_fp8_pull"], 2 * n, n + 4 * n_bs, copy_gbps)
    out["plain_e4m3_pull"] = entry(med["plain_e4m3_pull"], 2 * n, n, copy_gbps)

    exact = {}
    for key, gran, q, scales in (("channel_fp8_pull", "channel", qc, cs), ("tensor_fp8_pull", "tensor", qt, tsc)):
        sync, _, kw = forms[key]
        asyncio.run(sync.pull(handles, q, **kw))
        torch.cuda.synchronize()
        ok = True
        for k in names:
            want_q, want_s = torch_quantize(sd[k], gran)
            ok &= torch.equal(q[k].view(torch.uint8), want_q.view(torch.uint8)) and \
                torch.equal(scales[k].view(torch.int32), want_s.view(torch.int32))
            del want_q, want_s
        exact[gran] = bool(ok)
    out["bit_exact_vs_torch_cuda"] = exact
    out["params"] = n
    for sync, _, _ in forms.values():
        sync.close()
    asyncio.run(src.cleanup())
    print(json.dumps(out))
    assert all(exact.values()), f"scaled pull differs from the torch-CUDA rendering: {exact}"


if __name__ == "__main__":
    main()

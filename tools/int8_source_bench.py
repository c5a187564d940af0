"""Scaled INT8 sources on one GPU, the Llama-3-8B bf16 state dict's linear weights (wq wk wv wo w1 w2 w3) at N=1,
every int8 form alternated in the same run with its float8_e4m3fn twin (which moves the same bytes):
* ``refresh()`` of source-side int8 vs e4m3fn staging per granularity, for full-size weights and for FSDP(8)-style
  row shards (eight sources, their kernel times summed);
* the verbatim int8 pull vs the verbatim fp8 pull into destinations of the same granularity, and the raw int8 byte
  pull of the same staging;
* the int8 -> bf16 vs fp8 -> bf16 dequantising pulls.

    python tools/int8_source_bench.py [--reps 10] [--warmup 3]

Kernel times come from the plans' own start/done events, medians over warmed, repeated launches.  Alongside: the
card's name and power limit and its measured device-to-device copy rate (torch copy_ of 4 GiB).  Every int8 form is
then checked bit for bit at full size: the staging against the torch-CUDA rendering (int8_source_oracle), the
verbatim and raw pulls against the staging, and the dequantising pull against ``(q.float() * s).to(bf16)``.
Prints one JSON line.
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
from oracle.int8_source_oracle import scale_shape, torch_dequantize, torch_quantize  # noqa: E402
from tools.fp8_sync_bench import copy_rate, entry  # noqa: E402
from torchstore_b200 import _native  # noqa: E402
from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource  # noqa: E402
from torchstore_b200.transport.types import TensorSlice  # noqa: E402

LINEAR = {"wq", "wk", "wv", "wo", "w1", "w2", "w3"}
GRANULARITIES = ("block", "channel", "tensor")
FORMATS = (("int8", torch.int8), ("fp8", torch.float8_e4m3fn))
FSDP = 8


def fsdp_sources(sd: dict, gran: str, qdtype: torch.dtype) -> list:
    """FSDP(8)-style row shards of every weight, one quantising source per rank."""
    out = []
    for r in range(FSDP):
        shards, slices = {}, {}
        for k, v in sd.items():
            step = v.shape[0] // FSDP
            shards[k] = v[r * step:(r + 1) * step]
            slices[k] = TensorSlice((r * step, 0), (r,), tuple(v.shape), (step, v.shape[1]), (FSDP,))
        src = DirectWeightSyncSource()
        src.register(shards, rank=r, tensor_slices=slices, quantize={k: gran for k in sd}, quant_dtype=qdtype)
        out.append(src)
    return out


def refresh_ms(sources: list) -> float:
    for src in sources:
        src.refresh()
    return sum(sum(src._quant_plans.elapsed_ms().values()) for src in sources)


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
    n = sum(v.numel() for v in sd.values())
    exact = {}
    for gran in GRANULARITIES:
        n_s = sum(torch.Size(scale_shape(gran, tuple(v.shape))).numel() for v in sd.values())
        two = 2 if gran == "tensor" else 1  # per tensor, a refresh reads the weights twice (two passes)
        # (read, written) bytes of each form
        moved = {"refresh": (2 * n * two, n + 4 * n_s), "verbatim": (n + 4 * n_s, n + 4 * n_s),
                 "dequant": (n + 4 * n_s, 2 * n), "raw": (n, n)}
        res, ok = {}, {}
        src, handles = {}, {}
        for fmt, qdtype in FORMATS:
            src[fmt] = DirectWeightSyncSource()
            handles[fmt] = {k: [h] for k, h in src[fmt].register(sd, rank=0, quantize={k: gran for k in sd},
                                                                  quant_dtype=qdtype).items()}
        staging = {k: src["int8"]._quantized[k][:2] for k in names}

        def alternate(forms: dict, kind: dict) -> None:
            times = {k: [] for k in forms}
            for i in range(args.warmup + args.reps):
                for key, fn in forms.items():
                    t = fn()
                    if i >= args.warmup:
                        times[key].append(t)
            for key, ts in times.items():
                res[key] = entry(statistics.median(ts), *moved[kind[key]], copy_gbps)

        def pull_form(sync, h, dests, kw):
            def fn():
                asyncio.run(sync.pull(h, dests, **kw))
                return sync.last_pull_ms[0]
            return fn

        # refresh, full size
        alternate({f"refresh_{fmt}": (lambda fmt=fmt: refresh_ms([src[fmt]])) for fmt, _ in FORMATS},
                  {f"refresh_{fmt}": "refresh" for fmt, _ in FORMATS})
        ok["refresh"] = all(torch.equal(q, tq) and torch.equal(s.view(torch.int32), ts.reshape(s.shape).view(torch.int32))
                            for k, (q, s) in staging.items() for tq, ts in [torch_quantize(sd[k], gran)])

        # verbatim int8 vs verbatim fp8 vs the raw int8 bytes
        pulls = {}
        for fmt, qdtype in FORMATS:
            scales = {k: torch.empty(scale_shape(gran, tuple(v.shape)), device="cuda") for k, v in sd.items()}
            pulls[f"verbatim_{fmt}"] = (DirectWeightSyncDest(), handles[fmt],
                                        {k: torch.empty(v.shape, dtype=qdtype, device="cuda") for k, v in sd.items()},
                                        {f"{gran}_scales": scales, "verbatim": True})
        pulls["raw_int8_bytes"] = (DirectWeightSyncDest(), handles["int8"],
                                   {k: torch.empty(v.shape, dtype=torch.int8, device="cuda") for k, v in sd.items()}, {})
        alternate({k: pull_form(*v) for k, v in pulls.items()},
                  {"verbatim_int8": "verbatim", "verbatim_fp8": "verbatim", "raw_int8_bytes": "raw"})
        _, _, vq, vkw = pulls["verbatim_int8"]
        vs = vkw[f"{gran}_scales"]
        ok["verbatim"] = all(torch.equal(vq[k], q) and torch.equal(vs[k].view(torch.int32), s.reshape(vs[k].shape).view(torch.int32))
                             for k, (q, s) in staging.items())
        ok["raw_bytes"] = all(torch.equal(pulls["raw_int8_bytes"][2][k], q) for k, (q, _) in staging.items())
        for sync, *_ in pulls.values():
            sync.close()
        del pulls, vq, vkw, vs

        # int8 -> bf16 vs fp8 -> bf16
        pulls = {f"dequant_{fmt}_to_bf16": (DirectWeightSyncDest(), handles[fmt], {k: torch.empty_like(v) for k, v in sd.items()}, {})
                 for fmt, _ in FORMATS}
        alternate({k: pull_form(*v) for k, v in pulls.items()}, {k: "dequant" for k in pulls})
        dq = pulls["dequant_int8_to_bf16"][2]
        ok["dequant_to_bf16"] = all(torch.equal(dq[k].view(torch.int16),
                                                torch_dequantize(q, s, gran, dst=torch.bfloat16).view(torch.int16))
                                    for k, (q, s) in staging.items())
        for sync, *_ in pulls.values():
            sync.close()
        del pulls, dq, staging
        for fmt, _ in FORMATS:
            asyncio.run(src[fmt].cleanup())
        del src, handles
        torch.cuda.empty_cache()

        # refresh of FSDP(8)-style shards
        fsdp = {fmt: fsdp_sources(sd, gran, qdtype) for fmt, qdtype in FORMATS}
        alternate({f"refresh_fsdp8_{fmt}": (lambda fmt=fmt: refresh_ms(fsdp[fmt])) for fmt, _ in FORMATS},
                  {f"refresh_fsdp8_{fmt}": "refresh" for fmt, _ in FORMATS})
        ok["refresh_fsdp8"] = True
        for k in names:
            step = sd[k].shape[0] // FSDP
            for r, shard_src in enumerate(fsdp["int8"]):
                fq, fs, _ = shard_src._quantized[k]
                tq, ts = torch_quantize(sd[k][r * step:(r + 1) * step], gran, r * step, 0)
                ok["refresh_fsdp8"] &= torch.equal(fq, tq) and torch.equal(fs.view(torch.int32),
                                                                           ts.reshape(fs.shape).view(torch.int32))
        for fmt, _ in FORMATS:
            for shard_src in fsdp[fmt]:
                asyncio.run(shard_src.cleanup())
        del fsdp
        torch.cuda.empty_cache()

        for form, (i8, f8) in {"refresh": ("refresh_int8", "refresh_fp8"),
                               "refresh_fsdp8": ("refresh_fsdp8_int8", "refresh_fsdp8_fp8"),
                               "verbatim": ("verbatim_int8", "verbatim_fp8"),
                               "dequant_to_bf16": ("dequant_int8_to_bf16", "dequant_fp8_to_bf16")}.items():
            res[f"{form}_int8_over_fp8"] = round(res[i8]["kernel_ms"] / res[f8]["kernel_ms"], 4)
        out[gran] = res
        exact[gran] = {k: bool(v) for k, v in ok.items()}
    out["bit_exact_vs_torch_cuda"] = exact
    out["params"] = n
    print(json.dumps(out))
    assert all(all(v.values()) for v in exact.values()), f"an int8 form differs from the torch-CUDA rendering: {exact}"


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""bench.py -- weight-sync GB/s of a Llama-3-8B bf16 state_dict resharded FSDP(N) -> TP(N).

    python bench.py --gpus N --steps K --warmup W            (torchrun launches it for N > 1)
    python bench.py --impl reference ...                      (the reference's CPU path, oracle port)
    python bench.py --config {4,4p,2,3a,3b,5} ...             (the other BASELINE.json configs)

A "step" is ONE weight sync of the whole state_dict: every rank holds its FSDP Shard(0) source
shard and pulls its TP shard from all sources through the public API
(``ts.put_state_dict(direct_rdma=True)`` / ``ts.get_state_dict(direct_rdma=True)``), which runs one
persistent copy_rects launch per destination GPU.

  value   state_dict bytes * K / device time of K steps (CUDA events, max over ranks), inputs
          resident in HBM when the timed region starts
  e2e     the same through the same API with HOST inputs: every step copies the rank's new source
          weights from pinned host memory (H2D), refreshes/fences the source, pulls, and reads a
          result sample back (D2H); wall clock, barrier + synchronize on both sides, max over ranks
  roofline      algorithmic bytes per copy_rects launch / its average duration vs the measured peak
  cpu_baseline  the oracle's port of the reference's shm path (2 memcpy per byte) on the host cores

Parity inside the bench: every destination shard is compared BIT FOR BIT (torch.equal on the int16
view of the whole flat destination buffer, i.e. order-sensitive) with shards sliced from the same
seeded full tensors, after the first sync, after the timed steps and after the e2e steps, at every N;
an int32 ``arange`` tensor goes through the same path once ("bit-exact for index tensors").

Configs (BASELINE.json `configs`; the default, 4, is the headline the metric is quoted on):
  1    host tier plumbing: one process, 1 MiB fp32 tensor, LocalRankStrategy over POSIX shm, no GPU
  4    FSDP(N) -> TP(N), colocated ranks (every GPU is source and destination)
  4p   two disjoint groups: FSDP(N/2) on GPUs 0..N/2-1 -> TP(N/2) on GPUs N/2..N-1 (all bytes cross NVSwitch)
  2    one flat 4 GiB bf16 tensor (+ an int32 arange variant), GPU 0 -> GPU 1, same placement
  3a   FSDP(N) Shard(0) -> ONE replicated reader (rank 0 pulls the whole state dict)
  3b   FSDP(N) Shard(0) -> EVERY rank reads the whole state dict (P2P pulls; --allgather: NCCL route)
  5    store path: put_batch / get_batch of flat bf16 keys, key size swept 1 MiB .. 8 GiB
"""

from __future__ import annotations

import argparse
import asyncio
import json
import math
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import workloads  # noqa: E402

METRIC = "weight-sync GB/s (state_dict bytes / wall s)"
# H100 SXM data sheet: NVLink 4 moves 900 GB/s per GPU counting both directions, 450 GB/s each way.  The
# peer-copy rate reached on an H100 box has not been measured, so the NVLink roofline uses the nominal figure.
NVLINK_NOMINAL_GBPS = 450.0
# device-to-device copy of 4 GiB, read + write bytes over time (tools/hbm_copy_peak.py), measured on an
# H100 80GB HBM3 (SXM) at a 400 W power limit; the data sheet's 3.35 TB/s is for 700 W
HBM_COPY_MEASURED_GBPS = 3026.0
# --dump-outputs writes at most this many bytes in all (every rank together)
DUMP_BUDGET_BYTES = 64 << 20


# =================================================================================================
# helpers
# =================================================================================================
def load_peaks():
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(path):
        with open(path) as f:
            return json.load(f), "measured (MEASURED_PEAKS.json)"
    return {"hbm_gbs": HBM_COPY_MEASURED_GBPS}, "measured D2D copy peak (H100 80GB HBM3, 400 W power limit)"


class ClockSampler:
    """SM clock + throttle reasons sampled DURING the timed region (NVML every ~5 ms; falls back to
    `nvidia-smi -lms` when pynvml is unavailable)."""

    REASONS = {"hw_slowdown": 0x8, "hw_thermal_slowdown": 0x40, "sw_thermal_slowdown": 0x20, "sw_power_cap": 0x4}

    def __init__(self, device_index: int):
        self.device_index = device_index
        self.samples: list[tuple[float, int, float]] = []
        self.sm_max = None
        self._stop = threading.Event()
        self._thread = None
        self._nvml = None

    def start(self):
        try:
            import pynvml

            pynvml.nvmlInit()
            self._nvml = pynvml
            self._handle = pynvml.nvmlDeviceGetHandleByIndex(self.device_index)
            self.sm_max = float(pynvml.nvmlDeviceGetMaxClockInfo(self._handle, pynvml.NVML_CLOCK_SM))
        except Exception:
            self._nvml = None
        self._thread = threading.Thread(target=self._loop_nvml if self._nvml else self._loop_smi, daemon=True)
        self._thread.start()

    def _loop_nvml(self):
        nv = self._nvml
        while not self._stop.is_set():
            try:
                clk = float(nv.nvmlDeviceGetClockInfo(self._handle, nv.NVML_CLOCK_SM))
                try:
                    reasons = int(nv.nvmlDeviceGetCurrentClocksEventReasons(self._handle))
                except Exception:
                    reasons = int(nv.nvmlDeviceGetCurrentClocksThrottleReasons(self._handle))
                try:
                    power = nv.nvmlDeviceGetPowerUsage(self._handle) / 1000.0
                except Exception:
                    power = 0.0
                self.samples.append((clk, reasons, power))
            except Exception:
                pass
            time.sleep(0.004)

    def _loop_smi(self):
        fields = "clocks.sm,clocks.max.sm,power.draw"
        while not self._stop.is_set():
            try:
                out = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader,nounits", "-i",
                                      str(self.device_index)], capture_output=True, text=True, timeout=5).stdout
                parts = [p.strip() for p in out.strip().split(",")]
                self.samples.append((float(parts[0]), 0, float(parts[2])))
                self.sm_max = float(parts[1])
            except Exception:
                pass

    def stop(self) -> dict:
        self._stop.set()
        if self._thread is not None:
            self._thread.join(timeout=6)
        clocks = [c for c, _, _ in self.samples]
        bits = 0
        for _, r, _ in self.samples:
            bits |= r
        reasons = sorted(name for name, mask in self.REASONS.items() if bits & mask)
        return {"sm_mhz": statistics.median(clocks) if clocks else None, "sm_max_mhz": self.sm_max, "reasons": reasons,
                "samples": len(clocks), "power_w_max": max((p for _, _, p in self.samples), default=None),
                "source": "nvml" if self._nvml else "nvidia-smi"}


_REAL_STDOUT_FD = None


def capture_stdout():
    """Route everything libraries print to stdout (e.g. NCCL's version banner) to stderr, so that
    stdout carries exactly ONE line: the JSON result written by emit()."""
    global _REAL_STDOUT_FD
    if _REAL_STDOUT_FD is None:
        sys.stdout.flush()
        _REAL_STDOUT_FD = os.dup(1)
        os.dup2(2, 1)


def emit(obj):
    line = (json.dumps(obj) + "\n").encode()
    if _REAL_STDOUT_FD is None:
        sys.stdout.write(line.decode())
        sys.stdout.flush()
    else:
        sys.stdout.flush()
        os.write(_REAL_STDOUT_FD, line)


# =================================================================================================
# reference arm / cpu baseline: the oracle's port of the reference's shm path on the host
# =================================================================================================
def _available_ram() -> int:
    try:
        import psutil

        return int(psutil.virtual_memory().available)
    except Exception:
        return 64 << 30


def cpu_reference_run(n_ranks: int, steps: int, warmup: int, budget_s: float = 20.0, layers: int | None = None):
    """Time put_state_dict + get_state_dict of the reference's SharedMemory path, restated:
    put = every source shard copied into its shm segment (transport/shared_memory.py:373-374);
    get = every stored rectangle that intersects the wanted slice copied segment -> destination
    (shared_memory.py:473-476, client.py:284-314).  Byte movement by oracle/copy_rects_ref.c with
    all host threads; Python/RPC/pickle overhead of the real reference is NOT included (favours it;
    oracle/calibrate_port.py calibrates the port against the real reference).

    Workload: the Llama-3-8B FSDP(n)->TP(n) sync, all n source and n destination ranks emulated in
    one address space -- the FULL 291-tensor layout when host RAM allows (3 x 16 GB), else the first
    L transformer layers (said in `sample`).  Stability: buffers are first-touched by the same pinned
    worker threads that later copy them (every worker owns the same byte range every step, so its
    pages are NUMA-local, like a long-lived shm segment), and the reported time is the MEDIAN step."""
    import numpy as np

    from oracle import c_oracle
    from torchstore_b200 import _native  # struct definition only (no GPU call)

    try:
        cores = len(os.sched_getaffinity(0))
    except AttributeError:
        cores = os.cpu_count() or 1
    threads = min(cores, 256)
    full_layout = workloads.llama_layout(workloads.LLAMA3_8B)
    full_bytes = workloads.state_dict_bytes(full_layout)
    if layers is None:
        use_full = _available_ram() > 3 * full_bytes + (24 << 30)
        layout = full_layout if use_full else workloads.llama_layout(workloads.LLAMA3_8B, n_layers=4, with_embeddings=False)
    else:
        use_full = False
        layout = workloads.llama_layout(workloads.LLAMA3_8B, n_layers=layers, with_embeddings=False)
    sample_bytes = workloads.state_dict_bytes(layout)

    # source shards (rank-major), shm segments, destinations: np.empty => untouched pages
    src, seg, dst = {}, {}, {}
    for name, (shape, tp) in layout.items():
        for r in range(n_ranks):
            off, shp = workloads.shard_box(shape, n_ranks, r, ("S", 0)) if n_ranks > 1 else ((0,) * len(shape), shape)
            src[(name, r)] = np.empty(shp, dtype=np.uint16)
            seg[(name, r)] = np.empty(shp, dtype=np.uint16)
        for r in range(n_ranks):
            off, shp = workloads.shard_box(shape, n_ranks, r, tp) if n_ranks > 1 else ((0,) * len(shape), shape)
            dst[(name, r)] = np.empty(shp, dtype=np.uint16)

    def window(arr, index):
        ptr = arr.ctypes.data
        strides = arr.strides
        shape = []
        for (a, b), st in zip(index, strides):
            ptr += a * st
            shape.append(b - a)
        return ptr, shape, strides

    def rect(r, s_ptr, d_ptr, shape, s_strides, d_strides):
        r.src, r.dst, r.ndim = s_ptr, d_ptr, max(1, len(shape))
        for i in range(_native.TSB_MAX_DIMS):
            r.extent[i], r.src_stride[i], r.dst_stride[i] = 1, 0, 0
        for i, (e, ss, ds) in enumerate(zip(shape, s_strides, d_strides)):
            r.extent[i], r.src_stride[i], r.dst_stride[i] = e, ss, ds
        r.src_dtype = r.dst_dtype = _native.TSB_U16
        r.src_device = -1

    # fill the sources from a random template with the SAME rect order and thread partition as the
    # put below: the worker that will read a source page is the one that first touches it
    rng = np.random.default_rng(0)
    biggest = max(a.size for a in src.values())
    template = rng.integers(0, 65536, size=min(biggest, 1 << 26), dtype=np.uint16)
    keys = list(src)
    fill_rects = _native.make_rect_array(len(keys) * (1 + biggest // template.size))
    nfill = 0
    for i, k in enumerate(keys):
        flat = src[k].reshape(-1)
        shift = (i * 7919) % 4096
        for lo in range(0, flat.size, template.size - 4096):
            hi = min(flat.size, lo + template.size - 4096)
            rect(fill_rects[nfill], template.ctypes.data + 2 * shift, flat.ctypes.data + 2 * lo, [hi - lo], [2], [2])
            nfill += 1
    c_oracle.copy_rects(fill_rects, nfill, 0, threads, pin=True)

    put_list = [(src[k], seg[k]) for k in keys]
    put_rects = _native.make_rect_array(len(put_list))
    for i, (a, b) in enumerate(put_list):
        full = tuple((0, e) for e in a.shape)
        sp, shape, ss = window(a, full)
        dp, _, ds = window(b, full)
        rect(put_rects[i], sp, dp, shape, ss, ds)
    get_specs = []
    for drank in range(n_ranks):
        for name, srank, s_idx, d_idx, _exact in workloads.fsdp_to_tp_rects(layout, n_ranks, drank):
            get_specs.append((seg[(name, srank)], s_idx, dst[(name, drank)], d_idx))
    get_rects = _native.make_rect_array(len(get_specs))
    for i, (a, s_idx, b, d_idx) in enumerate(get_specs):
        sp, shape, ss = window(a, s_idx)
        dp, _, ds = window(b, d_idx)
        rect(get_rects[i], sp, dp, shape, ss, ds)

    def one_sync():
        c_oracle.copy_rects(put_rects, len(put_list), 0, threads, pin=True)
        c_oracle.copy_rects(get_rects, len(get_specs), 0, threads, pin=True)

    for _ in range(max(1, warmup)):  # also the first touch of seg/dst by their owning workers
        one_sync()
    # the baseline must be doing the real work: every destination rectangle equals its source slice
    checked = 0
    for drank in range(n_ranks):
        for name, srank, s_idx, d_idx, _exact in workloads.fsdp_to_tp_rects(layout, n_ranks, drank):
            if use_full and checked % 7:  # full layout: check every 7th rectangle (3 x 16 GB of compares otherwise)
                checked += 1
                continue
            checked += 1
            got = dst[(name, drank)][tuple(slice(a, b) for a, b in d_idx)]
            want = src[(name, srank)][tuple(slice(a, b) for a, b in s_idx)]
            if not np.array_equal(got, want):
                raise SystemExit(f"cpu reference port produced wrong bytes for {name} ({srank}->{drank})")
    times = []
    t_begin = time.perf_counter()
    while len(times) < steps and (time.perf_counter() - t_begin < budget_s or not times):
        t0 = time.perf_counter()
        one_sync()
        times.append(time.perf_counter() - t0)
    med = statistics.median(times)
    gbps = sample_bytes / med / 1e9
    what = "the full 291-tensor llama3-8b layout" if use_full else f"first {len(layout) // 9} transformer layers of llama3-8b"
    return {
        "value": gbps,
        "ms_per_step": med * 1e3,
        "ms_min": min(times) * 1e3,
        "ms_max": max(times) * 1e3,
        "steps": len(times),
        "cores": threads,
        "kind": "port",
        "full_layout": use_full,
        "sample_bytes": sample_bytes,
        # measured on the host CPU against the UNMODIFIED reference (oracle/calibrate_port.py):
        # the port moves bytes 1.3-2.6x faster than the reference's Python/pickle/asyncio path
        "port_over_reference": [1.3, 2.6],
        "sample": (f"{what} ({sample_bytes} B of bf16, {len(put_list)} put copies + {len(get_specs)} get rectangles) "
                   f"FSDP({n_ranks})->TP({n_ranks}), all ranks emulated in one process, median of {len(times)} syncs "
                   f"(min {min(times) * 1e3:.1f} / max {max(times) * 1e3:.1f} ms); byte movement = oracle/copy_rects_ref.c on "
                   f"{threads} pinned threads, pages first-touched by their owning thread; no Python/RPC/pickle cost"),
    }


def _gloo_worker(rank, port, n_ranks, layers, q):
    """One side of the reference's Gloo transport, restated (transport/gloo.py:436-513): a 2-rank gloo
    group between a client (rank 0) and a storage volume (rank 1); every tensor is ONE send/recv pair of
    a contiguous CPU tensor (slices are made contiguous first, :493-495)."""
    import numpy as np
    import torch
    import torch.distributed as dist

    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=2)
    layout = workloads.llama_layout(workloads.LLAMA3_8B, n_layers=layers, with_embeddings=False)
    torch.manual_seed(0)
    shards = {}
    for name, (shape, tp) in layout.items():
        for r in range(n_ranks):
            _, shp = workloads.shard_box(shape, n_ranks, r, ("S", 0)) if n_ranks > 1 else (None, shape)
            # client: the source shards; volume: the stored copies
            shards[(name, r)] = torch.empty(shp, dtype=torch.int16).random_() if rank == 0 else torch.empty(shp, dtype=torch.int16)
    rects = [(name, s, tuple(slice(a, b) for a, b in s_idx), tuple(b - a for a, b in s_idx))
             for d in range(n_ranks) for name, s, s_idx, _d_idx, _e in workloads.fsdp_to_tp_rects(layout, n_ranks, d)]
    times = []
    for it in range(3):
        dist.barrier()
        t0 = time.perf_counter()
        for t in shards.values():          # put: client -> volume, one send per shard (gloo.py:470-513)
            (dist.send(t, 1) if rank == 0 else dist.recv(t, 0))
        for name, s, idx, shp in rects:    # get: volume -> client, one contiguous rectangle per send
            if rank == 1:
                dist.send(shards[(name, s)][idx].contiguous(), 0)
            else:
                dist.recv(torch.empty(shp, dtype=torch.int16), 1)
        dist.barrier()
        times.append(time.perf_counter() - t0)
    if rank == 0:
        q.put((min(times[1:]), workloads.state_dict_bytes(layout), len(shards), len(rects)))
    dist.destroy_process_group()


def gloo_leg(n_ranks: int, layers: int = 2):
    """The Gloo half of the reference's CPU transports on a bounded sample (north_star: "POSIX-shm/Gloo
    CPU transport"): loopback TCP between two local processes, per-tensor send/recv."""
    import socket

    import torch.multiprocessing as mp

    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gloo_worker, args=(r, port, n_ranks, layers, q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        secs, nbytes, n_put, n_get = q.get(timeout=240)
    finally:
        for p in procs:
            p.join(60)
    return {"value": nbytes / secs / 1e9, "unit": "GB/s", "kind": "port",
            "sample": f"first {layers} transformer layers ({nbytes} B), FSDP({n_ranks})->TP({n_ranks}): {n_put} put sends + {n_get} get sends "
                      "over a 2-rank gloo group on loopback TCP (one client process, one volume process), best of 2 after warm-up"}


def run_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    res = cpu_reference_run(args.gpus, args.steps, args.warmup, budget_s=60.0)
    gloo = None
    if os.environ.get("TSB_BENCH_GLOO", "1") == "1":
        try:
            gloo = gloo_leg(args.gpus)
        except Exception as e:  # noqa: BLE001 -- a side measurement must not sink the arm
            gloo = {"unavailable": f"{type(e).__name__}: {e}"}
    layout = workloads.llama_layout()
    emit({
        "impl": "reference",
        "metric": METRIC,
        "value": res["value"],
        "unit": "GB/s",
        "n_gpus": args.gpus,
        "steps": res["steps"],
        "warmup": args.warmup,
        "ms_per_step": res["ms_per_step"],
        "higher_is_better": True,
        "scaling": "strong",
        "vs_baseline": None,
        "dtype": "bf16",
        "data": "synthetic",
        "config": {"workload": f"llama3-8b bf16 state_dict FSDP({args.gpus})->TP({args.gpus}) put_state_dict+get_state_dict, "
                               "reference SharedMemory path restated on host memory"
                               + ("" if res["full_layout"] else " (bounded sample)"),
                   "state_dict_bytes": workloads.state_dict_bytes(layout), "tensors": len(layout),
                   "parallelism": f"fsdp{args.gpus}->tp{args.gpus}", "ms_min": res["ms_min"], "ms_max": res["ms_max"]},
        "cpu_baseline": {"value": res["value"], "unit": "GB/s", "cores": res["cores"], "kind": res["kind"],
                         "sample": res["sample"], "port_over_reference": res["port_over_reference"], "gloo_transport": gloo},
        "e2e": {"value": res["value"], "unit": "GB/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    })


# =================================================================================================
# our arm: shared plumbing
# =================================================================================================
class Ctx:
    """Everything a config needs: ranks, device, collectives for timing, phase logging."""

    def __init__(self, args):
        import faulthandler

        import torch
        import torch.distributed as dist

        self.args = args
        self.torch, self.dist = torch, dist
        self.rank = int(os.environ.get("RANK", "0"))
        self.world = int(os.environ.get("WORLD_SIZE", "1"))
        self.local_rank = int(os.environ.get("LOCAL_RANK", "0"))
        # a hung collective / RPC must leave evidence: dump every thread's stack to stderr after the
        # watchdog period, repeatedly ... and must not hang the caller forever: hard deadline
        faulthandler.enable()
        faulthandler.dump_traceback_later(int(os.environ.get("TSB_BENCH_WATCHDOG_S", "90")), repeat=True, file=sys.stderr)
        deadline = float(os.environ.get("TSB_BENCH_DEADLINE_S", "480"))

        def _deadline():
            print(f"[bench r{self.rank}] deadline of {deadline:.0f}s exceeded; aborting", file=sys.stderr, flush=True)
            faulthandler.dump_traceback(file=sys.stderr)
            os._exit(3)

        self._timer = threading.Timer(deadline, _deadline)
        self._timer.daemon = True
        self._timer.start()
        self.t_start = time.perf_counter()
        if self.world != args.gpus:
            raise SystemExit(f"--gpus {args.gpus} but WORLD_SIZE={self.world}: launch with torchrun --nproc-per-node {args.gpus}")
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29517")
        os.environ.setdefault("RANK", "0")
        os.environ.setdefault("LOCAL_RANK", "0")
        os.environ.setdefault("WORLD_SIZE", "1")
        os.environ.setdefault("LOCAL_WORLD_SIZE", str(self.world))
        torch.cuda.set_device(self.local_rank)
        self.dev = torch.device("cuda", self.local_rank)
        # host threads of this rank live on the GPU's NUMA node: pinned staging memory is first-touched
        # there (e2e H2D at full PCIe rate on both sockets) and launches come from nearby cores
        from torchstore_b200 import numa

        self.numa = numa.bind_to_gpu_numa(self.local_rank) if os.environ.get("TSB_BENCH_NUMA", "1") == "1" else {"bound": False}
        if not os.environ.get("TSB_KEEP_NCCL_DEBUG"):
            os.environ["NCCL_DEBUG"] = "WARN"  # the version banner goes to stdout; keep stdout to ONE JSON line
        self.phase(f"init_process_group (numa: {self.numa})")
        dist.init_process_group("nccl", device_id=self.dev)
        from torchstore_b200 import _native

        _native.init()
        self.native = _native

    def phase(self, msg):
        if os.environ.get("TSB_BENCH_VERBOSE", "1") == "1":
            print(f"[bench r{self.rank} +{time.perf_counter() - self.t_start:7.2f}s] {msg}", file=sys.stderr, flush=True)

    def barrier(self):
        self.dist.barrier(device_ids=[self.local_rank])
        self.torch.cuda.synchronize()

    def allmax(self, x: float) -> float:
        t = self.torch.tensor([x], dtype=self.torch.float64, device=self.dev)
        self.dist.all_reduce(t, op=self.dist.ReduceOp.MAX)
        return float(t.item())

    def allsum(self, x: float) -> float:
        t = self.torch.tensor([x], dtype=self.torch.float64, device=self.dev)
        self.dist.all_reduce(t, op=self.dist.ReduceOp.SUM)
        return float(t.item())

    def gather_objects(self, obj):
        out = [None] * self.world
        self.dist.all_gather_object(out, obj)
        return out

    def done(self):
        import faulthandler

        faulthandler.cancel_dump_traceback_later()
        self._timer.cancel()


def build_shards(ctx: Ctx, layout, src_box, dst_box):
    """Seeded synthetic weights: for every tensor of `layout` the full tensor is generated on the GPU
    (same seed on every rank), `src_box(name, shape, tp)` / `dst_box(...)` -> (offsets, shape) or None
    select what this rank holds.  Returns flat parameter buffers (one allocation per side, like FSDP
    flat params), per-tensor views, and `expect_flat`: the destination buffer as it must look after a
    sync (same layout as dst_flat, zeros in the alignment slack)."""
    torch, dev = ctx.torch, ctx.dev
    boxes = {}
    src_numel = dst_numel = 0
    for name, (shape, tp) in layout.items():
        sb, db = src_box(name, shape, tp), dst_box(name, shape, tp)
        boxes[name] = (sb, db)
        if sb is not None:
            src_numel += (math.prod(sb[1]) + 63) // 64 * 64  # 128-byte aligned tensors
        if db is not None:
            dst_numel += (math.prod(db[1]) + 63) // 64 * 64
    src_flat = torch.empty(max(src_numel, 64), dtype=torch.bfloat16, device=dev)
    dst_flat = torch.zeros(max(dst_numel, 64), dtype=torch.bfloat16, device=dev)
    expect_flat = torch.zeros(max(dst_numel, 64), dtype=torch.bfloat16, device=dev)
    src_local, dst_local = {}, {}
    so = do = 0
    gen = torch.Generator(device=dev)
    for idx, (name, (shape, tp)) in enumerate(layout.items()):
        sb, db = boxes[name]
        if sb is None and db is None:
            continue
        gen.manual_seed(1234 + idx)
        full = (torch.randn(shape, generator=gen, device=dev, dtype=torch.float32) * 0.02).to(torch.bfloat16)
        if sb is not None:
            ns = math.prod(sb[1])
            src_local[name] = src_flat[so:so + ns].view(sb[1])
            src_local[name].copy_(full[tuple(slice(o, o + e) for o, e in zip(*sb))])
            so += (ns + 63) // 64 * 64
        if db is not None:
            nd = math.prod(db[1])
            dst_local[name] = dst_flat[do:do + nd].view(db[1])
            expect_flat[do:do + nd].view(db[1]).copy_(full[tuple(slice(o, o + e) for o, e in zip(*db))])
            do += (nd + 63) // 64 * 64
        del full
    torch.cuda.synchronize()
    return dict(boxes=boxes, src_flat=src_flat, dst_flat=dst_flat, expect_flat=expect_flat, src=src_local, dst=dst_local)


def verify_flat(ctx: Ctx, sh, tag: str):
    """Order-sensitive, bit-exact: the whole flat destination buffer against the expected one."""
    torch = ctx.torch
    got, want = sh["dst_flat"].view(torch.int16), sh["expect_flat"].view(torch.int16)
    if not torch.equal(got, want):
        bad = []
        for name, v in sh["dst"].items():
            off = (v.data_ptr() - sh["dst_flat"].data_ptr()) // 2
            if not torch.equal(got[off:off + v.numel()], want[off:off + v.numel()]):
                bad.append(name)
        raise SystemExit(f"[rank {ctx.rank}] PARITY FAILURE after {tag}: {bad[:5]} ({len(bad)} tensors differ bitwise)")


def dump_outputs(ctx: Ctx, tensors: dict, out_dir: str):
    """Write what the timed path delivered: every destination tensor as DIR/<name>.npy in float32
    (rank<r>.<name>.npy when N > 1).  A tensor larger than its share of the budget is sampled at a
    fixed, seeded set of element positions, so two builds run with the same arguments can be compared
    file for file."""
    import numpy as np

    torch = ctx.torch
    os.makedirs(out_dir, exist_ok=True)
    header = 128  # .npy header of a 1-D array
    per_tensor = (DUMP_BUDGET_BYTES // ctx.world // max(1, len(tensors)) - header) // 4
    prefix = f"rank{ctx.rank}." if ctx.world > 1 else ""
    for i, (name, t) in enumerate(tensors.items()):
        flat = t.reshape(-1)
        if flat.numel() > per_tensor:
            gen = torch.Generator().manual_seed(i)
            idx = torch.randint(0, flat.numel(), (per_tensor,), generator=gen).sort().values
            flat = flat[idx.to(flat.device)]
        np.save(os.path.join(out_dir, f"{prefix}{name}.npy"), flat.float().cpu().numpy())


def full_box(name, shape, tp):
    return (0,) * len(shape), tuple(shape)


async def timed_steps(ctx: Ctx, step, kernel_ms_of, zero=None):
    """W warm-up steps, then exactly K steps bracketed by barrier + synchronize; device time from
    CUDA events on the copy stream (the stream copy_rects is launched on), max over ranks."""
    args, native = ctx.args, ctx.native
    for _ in range(args.warmup):
        await step()
        ctx.barrier()
    if zero is not None:
        zero()
    ctx.barrier()
    sampler = ClockSampler(ctx.local_rank)
    if ctx.rank == 0:
        sampler.start()
    launches0 = native.launch_count()
    kernel_ms = []
    copy_stream = native.copy_stream(ctx.local_rank)
    ev0 = native.Event(ctx.local_rank, timing=True)
    ev1 = native.Event(ctx.local_rank, timing=True)
    ctx.barrier()
    if args.profiler_range:
        ctx.torch.cuda.cudart().cudaProfilerStart()
    ev0.record(copy_stream)
    t0 = time.perf_counter()
    for _ in range(args.steps):
        # K syncs back to back on every rank; the bracket is barrier + synchronize on both sides.
        # (The cross-rank "sources are ready" dependency of a real sync is part of the e2e leg.)
        await step()
        k = kernel_ms_of()
        if k is not None:
            kernel_ms.append(k)
    ev1.record(copy_stream)
    ev1.synchronize()
    wall_ms = (time.perf_counter() - t0) * 1e3
    if args.profiler_range:
        ctx.torch.cuda.cudart().cudaProfilerStop()
    dev_ms = ev0.elapsed_ms(ev1)
    ctx.phase(f"timed steps done: {dev_ms / args.steps:.3f} ms/step on this rank")
    ctx.barrier()
    launches = native.launch_count() - launches0
    clocks = sampler.stop() if ctx.rank == 0 else None
    kern_avg = sum(kernel_ms) / len(kernel_ms) if kernel_ms else 0.0
    return dict(dev_ms=ctx.allmax(dev_ms), wall_ms=ctx.allmax(wall_ms), kern_avg=ctx.allmax(kern_avg),
                launches=int(ctx.allsum(launches)), clocks=clocks)


def roofline_for(n_remote_bound: bool, info, kern_ms):
    """HBM-bound launches: bytes read locally + bytes written, vs the measured HBM copy peak.
    NVLink-bound launches: bytes pulled from peers vs the nominal per-direction NVLink rate.
    `traffic` (DRAM bytes counted by the hardware) is not measured: null."""
    peaks, peak_src = load_peaks()
    local_read = info["src_bytes"] - info["remote_src_bytes"]
    algo_hbm = local_read + info["payload_bytes"]
    kern_s = max(kern_ms, 1e-9) / 1e3
    if not n_remote_bound:
        return {"bound": "hbm", "achieved": algo_hbm / kern_s / 1e9, "peak": peaks["hbm_gbs"], "unit": "GB/s",
                "frac": algo_hbm / kern_s / 1e9 / peaks["hbm_gbs"], "traffic": None, "traffic_source": "not measured",
                "peak_source": peak_src, "kernel": "copy_rects_kernel<KIND_B16>",
                "algorithmic_bytes_per_launch": algo_hbm, "kernel_ms_avg": kern_ms}
    nvl = info["remote_src_bytes"] / kern_s / 1e9
    # this GPU's HBM also serves the peers' reads of its shards (symmetric plans: as many bytes out as in)
    hbm_bytes = algo_hbm + info["remote_src_bytes"]
    return {"bound": "nvlink", "achieved": nvl, "peak": NVLINK_NOMINAL_GBPS, "unit": "GB/s",
            "frac": nvl / NVLINK_NOMINAL_GBPS, "traffic": None, "nvlink_traffic": None, "traffic_source": "not measured",
            "peak_source": "nominal NVLink 4 per direction (H100 SXM data sheet); peer-copy rate not measured",
            "kernel": "copy_rects_kernel<KIND_B16> (copy warps: local HBM; link warp: TMA bulk over NVLink)",
            "algorithmic_bytes_per_launch": info["remote_src_bytes"], "kernel_ms_avg": kern_ms,
            "hbm": {"achieved": hbm_bytes / kern_s / 1e9, "peak": peaks["hbm_gbs"],
                    "frac": hbm_bytes / kern_s / 1e9 / peaks["hbm_gbs"],
                    "algorithmic_bytes_per_launch_incl_serving_peers": hbm_bytes}}


def base_line(ctx: Ctx, value, ms_per_step, workload, extra_config, timed, roofline, e2e, cpu, nvlink_fraction, scaling="strong"):
    return {
        "metric": METRIC,
        "value": value,
        "unit": "GB/s",
        "n_gpus": ctx.world,
        "steps": ctx.args.steps,
        "warmup": ctx.args.warmup,
        "ms_per_step": ms_per_step,
        "higher_is_better": True,
        "scaling": scaling,
        "vs_baseline": None,
        "dtype": "bf16",
        "data": "synthetic",
        "config": {"workload": workload, "bench_config": ctx.args.config,
                   "l2": "inputs larger than L2 (>= 2 GB moved per GPU per step; no flush)", "numa": ctx.numa, **extra_config},
        "clocks": timed["clocks"],
        "e2e": e2e,
        "gpu_launches": timed["launches"],
        "roofline": roofline,
        "nvlink_fraction": nvlink_fraction,
        "cpu_baseline": None if cpu is None else {"value": cpu["value"], "unit": "GB/s", "cores": cpu["cores"], "kind": cpu["kind"],
                                                  "sample": cpu["sample"], "port_over_reference": cpu["port_over_reference"]},
    }


def dtensor_dict(ctx: Ctx, local, layout, placement_of):
    """Plain local shards -> DTensors on the 1-D mesh over all ranks (what FSDP / TP hand the API)."""
    torch = ctx.torch
    if ctx.world == 1:
        return dict(local)
    from torch.distributed.device_mesh import init_device_mesh
    from torch.distributed.tensor import DTensor, Replicate, Shard

    if not hasattr(ctx, "mesh"):
        ctx.mesh = init_device_mesh("cuda", (ctx.world,))

    def P(p):
        return Shard(p[1]) if p[0] == "S" else Replicate()

    return {k: DTensor.from_local(v, ctx.mesh, (P(placement_of(k)),), run_check=False, shape=torch.Size(layout[k][0]),
                                  stride=torch.empty(layout[k][0], device="meta").stride())
            for k, v in local.items()}


async def init_store(ctx: Ctx):
    import torchstore_b200 as ts

    if ctx.world > 1:
        # reuse the process group's c10d store as the rendezvous (no second TCP server)
        await ts.initialize_spmd(ts.LocalRankStrategy(), rendezvous=ctx.dist.distributed_c10d._get_default_store())
    else:
        await ts.initialize()
    ctx.phase("store initialized")
    return ts


# =================================================================================================
# config 4 (headline): FSDP(N) -> TP(N), colocated ranks
# =================================================================================================
async def cfg_headline(ctx: Ctx):
    torch, native, args = ctx.torch, ctx.native, ctx.args
    n, rank = ctx.world, ctx.rank
    from torchstore_b200.planner import StridedMem, build_rects

    layout = workloads.llama_layout(workloads.LLAMA3_8B)
    sd_bytes = workloads.state_dict_bytes(layout)
    ctx.phase("generating weights")

    def src_box(name, shape, tp):
        return workloads.shard_box(shape, n, rank, ("S", 0)) if n > 1 else full_box(name, shape, tp)

    def dst_box(name, shape, tp):
        return workloads.shard_box(shape, n, rank, tp) if n > 1 else full_box(name, shape, tp)

    sh = build_shards(ctx, layout, src_box, dst_box)
    src_flat, dst_flat = sh["src_flat"], sh["dst_flat"]
    ctx.phase("weights ready")
    src_sd = dtensor_dict(ctx, sh["src"], layout, lambda k: ("S", 0))
    dst_sd = dtensor_dict(ctx, sh["dst"], layout, lambda k: layout[k][1])
    ctx.phase("state dicts wrapped (DTensors on the 1-D mesh)")
    ts = await init_store(ctx)
    KEY = "policy"

    # first sync: registers handles, exchanges them through the store, builds + caches the plan
    t_first = time.perf_counter()
    await ts.put_state_dict(src_sd, KEY, direct_rdma=True)
    ctx.phase("handles published")
    ctx.barrier()
    await ts.get_state_dict(KEY, user_state_dict=dst_sd, direct_rdma=True)
    ctx.phase("first pull done")
    ctx.barrier()
    first_ms = (time.perf_counter() - t_first) * 1e3
    verify_flat(ctx, sh, "first sync")
    ctx.phase("first sync verified (bit-exact, order-sensitive)")

    # ---- index tensors: an int32 arange goes through the same path once, bit-exact -----------------
    ishape = (4096, 8192)
    ilayout = {"index.weight": (ishape, ("S", 1))}
    ifull = torch.arange(ishape[0] * ishape[1], dtype=torch.int32, device=ctx.dev).view(ishape)
    ib = (workloads.shard_box(ishape, n, rank, ("S", 0)), workloads.shard_box(ishape, n, rank, ("S", 1))) if n > 1 else \
        (full_box(None, ishape, None), full_box(None, ishape, None))
    isrc = ifull[tuple(slice(o, o + e) for o, e in zip(*ib[0]))].contiguous()
    iwant = ifull[tuple(slice(o, o + e) for o, e in zip(*ib[1]))].contiguous()
    idst = torch.zeros_like(iwant)
    await ts.put_state_dict(dtensor_dict(ctx, {"index.weight": isrc}, ilayout, lambda k: ("S", 0)), "index_check", direct_rdma=True)
    ctx.barrier()
    await ts.get_state_dict("index_check", user_state_dict=dtensor_dict(ctx, {"index.weight": idst}, ilayout, lambda k: ("S", 1)),
                            direct_rdma=True)
    if not torch.equal(idst, iwant):
        raise SystemExit(f"[rank {rank}] PARITY FAILURE: int32 arange tensor not bit-exact after reshard")
    ctx.barrier()
    del ifull, isrc, iwant, idst
    ctx.phase("int32 index tensor verified")

    from torchstore_b200.state_dict_utils import _get_rdma_cache

    cl = await ts.client()
    dest_sync = _get_rdma_cache(cl).dests[KEY]
    info = dest_sync.plan_info()[ctx.local_rank]

    async def step():
        await ts.put_state_dict(None, KEY, direct_rdma=True)  # refresh + fence on the source side
        await ts.get_state_dict(KEY, user_state_dict=dst_sd, direct_rdma=True)

    timed = await timed_steps(ctx, step, lambda: dest_sync.last_pull_ms[ctx.local_rank], zero=lambda: dst_flat.zero_())
    verify_flat(ctx, sh, "timed steps")
    if args.dump_outputs:
        dump_outputs(ctx, sh["dst"], args.dump_outputs)
    if rank == 0 and os.environ.get("TSB_BENCH_LIST_CONTEXTS"):
        # evidence that no rank holds a stray CUDA context on another rank's GPU (round-1 DeviceGuard bug)
        try:
            out = subprocess.run(["nvidia-smi", "--query-compute-apps=pid,gpu_bus_id,used_memory", "--format=csv,noheader"],
                                 capture_output=True, text=True, timeout=20).stdout
            ctx.phase("compute contexts per GPU (pid, bus id, memory):\n" + out)
        except Exception as e:  # noqa: BLE001
            ctx.phase(f"nvidia-smi failed: {e}")

    # development hook (not part of the contract line): TSB_BENCH_SWEEP="K=V,K=V;K=V;..." re-plans the same sync
    # under each launch setting and times it in place, so one multi-GPU job compares many settings
    sweep_rows = []
    if os.environ.get("TSB_BENCH_SWEEP"):
        for setting in os.environ["TSB_BENCH_SWEEP"].split(";"):
            saved = {}
            for kv in filter(None, setting.split(",")):
                k, v = kv.split("=")
                saved[k] = os.environ.get(k)
                os.environ[k] = v
            dest_sync.close()  # plan_create reads the launch settings; the next pull re-plans
            ctx.barrier()
            for _ in range(3):
                await step()
            dst_flat.zero_()
            ctx.barrier()
            ks = []
            t0 = time.perf_counter()
            for _ in range(args.steps):
                await step()
                ks.append(dest_sync.last_pull_ms[ctx.local_rank])
            wall = (time.perf_counter() - t0) * 1e3 / args.steps
            ctx.barrier()
            verify_flat(ctx, sh, f"sweep {setting}")
            row = {"env": setting, "kernel_ms_avg_max_rank": ctx.allmax(sum(ks) / len(ks)), "wall_ms_per_step_max_rank": ctx.allmax(wall),
                   "kernel_ms_min_over_steps_max_rank": ctx.allmax(min(ks))}
            sweep_rows.append(row)
            ctx.phase(f"sweep {setting or '(defaults)'}: kernel {row['kernel_ms_avg_max_rank']:.4f} ms, wall {row['wall_ms_per_step_max_rank']:.4f} ms")
            for k, v in saved.items():
                if v is None:
                    os.environ.pop(k, None)
                else:
                    os.environ[k] = v
        dest_sync.close()
        await step()

    e2e_ms, e2e_launches, src_bytes, d2h_bytes, h2d_gbps = None, 0, 0, 0, None
    if not args.no_e2e:
        # ---- e2e: host inputs, public API, wall clock ------------------------------------------------
        from torchstore_b200 import numa

        src_bytes = src_flat.numel() * 2
        host_src = numa.pinned_like(src_bytes, torch.bfloat16)  # first-touched on the GPU's NUMA node, then page-locked
        copy_stream = native.copy_stream(ctx.local_rank)
        native.memcpy_async(ctx.local_rank, host_src.data_ptr(), src_flat.data_ptr(), src_bytes, native.TSB_D2H, copy_stream)
        native.stream_sync(ctx.local_rank, copy_stream)
        # result sample: first row (<= 4096 elements) of every destination tensor, gathered by one
        # copy_rects launch into a contiguous buffer and read back with one D2H copy
        rows = []
        for k, v in sh["dst"].items():
            flat = v.reshape(-1) if v.dim() == 1 else v[0]
            rows.append(flat[: min(4096, flat.numel())])
        sample_dev = torch.zeros(sum(r.numel() for r in rows), dtype=torch.bfloat16, device=ctx.dev)
        pairs, off = [], 0
        for r in rows:
            pairs.append((StridedMem.from_tensor(r), StridedMem.from_tensor(sample_dev[off:off + r.numel()])))
            off += r.numel()
        rects, nr = build_rects(pairs)
        sample_plan = native.plan_create(ctx.local_rank, rects, nr)
        d2h_bytes = sample_dev.numel() * 2
        sample_host = numa.pinned_like(d2h_bytes, torch.bfloat16)
        h2d_ms = []

        async def e2e_step():
            # (1) new weights arrive from the host
            t0 = time.perf_counter()
            native.memcpy_async(ctx.local_rank, src_flat.data_ptr(), host_src.data_ptr(), src_bytes, native.TSB_H2D, copy_stream)
            native.stream_sync(ctx.local_rank, copy_stream)
            h2d_ms.append((time.perf_counter() - t0) * 1e3)
            # (2) publish + pull through the public API
            await ts.put_state_dict(None, KEY, direct_rdma=True)
            if n > 1:
                ctx.dist.barrier(device_ids=[ctx.local_rank])  # every source refreshed before anyone pulls
            await ts.get_state_dict(KEY, user_state_dict=dst_sd, direct_rdma=True)
            # (3) read the result sample back
            native.plan_run(sample_plan, copy_stream)
            native.memcpy_async(ctx.local_rank, sample_host.data_ptr(), sample_dev.data_ptr(), d2h_bytes, native.TSB_D2H, copy_stream)
            native.stream_sync(ctx.local_rank, copy_stream)

        for _ in range(max(1, min(args.warmup, 2))):
            await e2e_step()
        dst_flat.zero_()
        h2d_ms.clear()
        ctx.barrier()
        e_launch0 = native.launch_count()
        t0 = time.perf_counter()
        for _ in range(args.steps):
            await e2e_step()
        ctx.barrier()
        ctx.phase("e2e steps done")
        e2e_ms = ctx.allmax((time.perf_counter() - t0) * 1e3)
        e2e_launches = int(ctx.allsum(native.launch_count() - e_launch0))
        h2d_gbps = src_bytes / (ctx.allmax(statistics.median(h2d_ms)) / 1e3) / 1e9  # slowest rank's median H2D rate
        assert torch.equal(sample_host.to(ctx.dev), sample_dev)
        verify_flat(ctx, sh, "e2e steps")
        native.plan_destroy(sample_plan)
        native.host_unregister(host_src.data_ptr())
        native.host_unregister(sample_host.data_ptr())
    h2d_total, d2h_total = int(ctx.allsum(src_bytes)), int(ctx.allsum(d2h_bytes))

    cpu = None
    if rank == 0 and n == 1 and not args.no_cpu_baseline:
        cpu = cpu_reference_run(1, steps=1000, warmup=1, budget_s=15.0)
    if rank != 0:
        return None
    steps = args.steps
    value = sd_bytes * steps / (timed["dev_ms"] / 1e3) / 1e9
    e2e = sd_bytes * steps / (e2e_ms / 1e3) / 1e9 if e2e_ms else None
    roofline = roofline_for(n > 1, info, timed["kern_avg"])
    return base_line(
        ctx, value, timed["dev_ms"] / steps,
        f"llama3-8b bf16 state_dict ({len(layout)} tensors) FSDP({n}) Shard(0) -> TP({n}) direct_weight_sync via "
        "ts.put_state_dict/get_state_dict(direct_rdma=True), colocated ranks",
        {"state_dict_bytes": sd_bytes, "parallelism": f"fsdp{n}->tp{n}", "rects_per_dest_rank": info["num_rects"],
         "tiles_per_launch": info["num_tiles"], "link_tiles_per_launch": info["num_link_tiles"], "grid": info["grid"],
         "block": info["block"], "first_sync_ms_incl_registration_and_planning": first_ms,
         "wall_ms_per_step": timed["wall_ms"] / steps,
         "host_overhead_ms_per_step": timed["wall_ms"] / steps - timed["kern_avg"],
         "parity": "bit-exact torch.equal of every destination shard (order-sensitive) after first sync, timed steps and e2e; "
                   "int32 arange tensor bit-exact", **({"launch_setting_sweep": sweep_rows} if sweep_rows else {})},
        timed, roofline,
        {"value": e2e, "unit": "GB/s", "h2d_bytes_per_step": h2d_total, "d2h_bytes_per_step": d2h_total,
         "ms_per_step": (e2e_ms / steps) if e2e_ms else None, "gpu_launches": e2e_launches,
         "h2d_GBps_per_gpu_slowest_rank": h2d_gbps},
        cpu, (info["remote_src_bytes"] / (timed["dev_ms"] / steps / 1e3) / 1e9 / NVLINK_NOMINAL_GBPS) if n > 1 else 0.0)


# =================================================================================================
# low-level direct sync between explicit source / destination rank sets (configs 4p and 2)
# =================================================================================================
async def direct_sync(ctx: Ctx, ts, key, src_index, n_src, src_tensors, src_slices, dst_tensors, dst_slices):
    """Publish handles from the source ranks (ts.put), collect them on the destination ranks (ts.get),
    first pull.  Returns (source or None, dest or None, all_handles)."""
    from torchstore_b200.direct_weight_sync import DirectWeightSyncDest, DirectWeightSyncSource

    source = dest = all_handles = None
    if src_tensors:
        source = DirectWeightSyncSource()
        handles = source.register(src_tensors, rank=src_index, tensor_slices=src_slices)
        await ts.put(f"{key}/rank_{src_index}", handles)
    ctx.barrier()
    if dst_tensors:
        all_handles = {}
        for r in range(n_src):
            for name, h in (await ts.get(f"{key}/rank_{r}")).items():
                all_handles.setdefault(name, []).append(h)
        dest = DirectWeightSyncDest()
        await dest.pull(all_handles, dst_tensors, dst_slices)
    ctx.barrier()
    return source, dest, all_handles


def pick_info(ctx: Ctx, dest):
    infos = ctx.gather_objects(dest.plan_info()[ctx.local_rank] if dest is not None else None)
    return next(i for i in infos if i is not None)


async def cfg_disjoint(ctx: Ctx):
    """Config #4 as literally stated: two disjoint actor groups.  FSDP(N/2) on GPUs 0..N/2-1 ->
    TP(N/2) on GPUs N/2..N-1: every byte crosses NVSwitch, N/2 x 4 GB (N=8) into each destination."""
    torch, args = ctx.torch, ctx.args
    n, rank = ctx.world, ctx.rank
    if n < 2 or n % 2:
        raise SystemExit("--config 4p needs an even number of GPUs >= 2")
    from torchstore_b200.transport.types import TensorSlice

    half = n // 2
    is_src = rank < half
    g = rank if is_src else rank - half
    layout = workloads.llama_layout(workloads.LLAMA3_8B)
    sd_bytes = workloads.state_dict_bytes(layout)

    def sbox(name, shape, tp):
        if not is_src:
            return None
        return workloads.shard_box(shape, half, g, ("S", 0)) if half > 1 else full_box(name, shape, tp)

    def dbox(name, shape, tp):
        if is_src:
            return None
        return workloads.shard_box(shape, half, g, tp) if half > 1 else full_box(name, shape, tp)

    sh = build_shards(ctx, layout, sbox, dbox)
    ctx.phase("weights ready")

    def slices(which):
        out = {}
        for name, (sb, db) in sh["boxes"].items():
            b = sb if which == "src" else db
            if b is not None:
                out[name] = TensorSlice(tuple(b[0]), (g,), tuple(layout[name][0]), tuple(b[1]), (half,))
        return out

    ts = await init_store(ctx)
    t_first = time.perf_counter()
    source, dest, all_handles = await direct_sync(ctx, ts, "policy4p", g, half, sh["src"], slices("src"), sh["dst"], slices("dst"))
    first_ms = (time.perf_counter() - t_first) * 1e3
    dst_slices = slices("dst")
    if dest is not None:
        verify_flat(ctx, sh, "first sync")
    info = pick_info(ctx, dest)

    async def step():
        if source is not None:
            source.refresh()
            source.fence()
        if dest is not None:
            await dest.pull(all_handles, sh["dst"], dst_slices)

    timed = await timed_steps(ctx, step, (lambda: dest.last_pull_ms[ctx.local_rank]) if dest is not None else (lambda: None),
                              zero=lambda: sh["dst_flat"].zero_())
    if dest is not None:
        verify_flat(ctx, sh, "timed steps")
    ctx.barrier()
    if rank != 0:
        return None
    steps = args.steps
    value = sd_bytes * steps / (timed["dev_ms"] / 1e3) / 1e9
    roofline = roofline_for(True, info, timed["kern_avg"])
    return base_line(
        ctx, value, timed["dev_ms"] / steps,
        f"llama3-8b bf16 state_dict FSDP({half}) on GPUs 0..{half - 1} -> TP({half}) on GPUs {half}..{n - 1} "
        "(disjoint groups, every byte crosses NVSwitch), DirectWeightSyncSource/Dest + ts.put/ts.get of the handles",
        {"state_dict_bytes": sd_bytes, "parallelism": f"fsdp{half}->tp{half} disjoint", "rects_per_dest_rank": info["num_rects"],
         "link_tiles_per_launch": info["num_link_tiles"], "tiles_per_launch": info["num_tiles"],
         "bytes_into_each_dest_gpu": info["payload_bytes"], "first_sync_ms_incl_registration_and_planning": first_ms,
         "wall_ms_per_step": timed["wall_ms"] / steps, "parity": "bit-exact torch.equal of every destination shard"},
        timed, roofline, None, None, info["remote_src_bytes"] / (timed["dev_ms"] / steps / 1e3) / 1e9 / NVLINK_NOMINAL_GBPS)


async def cfg_flat2(ctx: Ctx):
    """Config #2: one flat 4 GiB bf16 tensor, GPU 0 -> GPU 1, same placement (a single exact-match op);
    then the int32 arange variant ("bit-exact for integer/index tensors")."""
    torch, args = ctx.torch, ctx.args
    n, rank = ctx.world, ctx.rank
    if n != 2:
        raise SystemExit("--config 2 needs exactly 2 GPUs")
    nbytes = 4 << 30
    ts = await init_store(ctx)
    results = {}
    for label, dtype in (("bf16", torch.bfloat16), ("int32", torch.int32)):
        numel = nbytes // dtype.itemsize
        if dtype == torch.int32:
            full = torch.arange(numel, dtype=torch.int32, device=ctx.dev)
        else:
            gen = torch.Generator(device=ctx.dev)
            gen.manual_seed(7)
            full = torch.empty(numel, dtype=dtype, device=ctx.dev)
            full.view(torch.int16).random_(-32768, 32767, generator=gen)  # arbitrary bit patterns, NaN payloads included
        dst = torch.zeros(numel, dtype=dtype, device=ctx.dev) if rank == 1 else None
        source, dest, all_handles = await direct_sync(ctx, ts, f"flat_{label}", 0, 1, {"flat": full} if rank == 0 else None, None,
                                                      {"flat": dst} if rank == 1 else None, None)

        def check(tag):
            if rank == 1 and not torch.equal(dst.view(torch.int16), full.view(torch.int16)):
                raise SystemExit(f"PARITY FAILURE ({label}) after {tag}")

        check("first sync")
        info = pick_info(ctx, dest)

        async def step():
            if source is not None:
                source.refresh()
                source.fence()
            if dest is not None:
                await dest.pull(all_handles, {"flat": dst})

        timed = await timed_steps(ctx, step, (lambda: dest.last_pull_ms[ctx.local_rank]) if dest is not None else (lambda: None),
                                  zero=(lambda: dst.zero_()) if dst is not None else None)
        check("timed steps")
        results[label] = (timed, info)
        if dest is not None:
            dest.close()
        if source is not None:
            await source.cleanup()
        del full, dst
        ctx.barrier()
    if rank != 0:
        return None
    steps = args.steps
    timed, info = results["bf16"]
    itimed, _ = results["int32"]
    value = nbytes * steps / (timed["dev_ms"] / 1e3) / 1e9
    roofline = roofline_for(True, info, timed["kern_avg"])
    return base_line(
        ctx, value, timed["dev_ms"] / steps,
        "direct_weight_sync of one flat 4 GiB bf16 tensor GPU0 -> GPU1, same placement (single exact-match op)",
        {"bytes": nbytes, "link_tiles_per_launch": info["num_link_tiles"], "tiles_per_launch": info["num_tiles"],
         "wall_ms_per_step": timed["wall_ms"] / steps,
         "int32_arange_variant": {"GBps": nbytes * steps / (itimed["dev_ms"] / 1e3) / 1e9, "kernel_ms_avg": itimed["kern_avg"],
                                  "parity": "bit-exact"},
         "parity": "bit-exact (torch.equal on the raw 16-bit patterns, NaN payloads included)"},
        timed, roofline, None, None, nbytes / (timed["dev_ms"] / steps / 1e3) / 1e9 / NVLINK_NOMINAL_GBPS)


# =================================================================================================
# config 3: FSDP(N) Shard(0) -> replicated reader(s)
# =================================================================================================
async def cfg_replicated(ctx: Ctx, all_readers: bool):
    torch, args = ctx.torch, ctx.args
    n, rank = ctx.world, ctx.rank
    if args.allgather:
        os.environ["TORCHSTORE_B200_ALLGATHER"] = "1"
    layout = workloads.llama_layout(workloads.LLAMA3_8B)
    sd_bytes = workloads.state_dict_bytes(layout)
    reader = all_readers or rank == 0

    def sbox(name, shape, tp):
        return workloads.shard_box(shape, n, rank, ("S", 0)) if n > 1 else full_box(name, shape, tp)

    sh = build_shards(ctx, layout, sbox, full_box if reader else (lambda *a: None))
    ctx.phase("weights ready")
    src_sd = dtensor_dict(ctx, sh["src"], layout, lambda k: ("S", 0))
    ts = await init_store(ctx)
    KEY = "policy3"
    t_first = time.perf_counter()
    await ts.put_state_dict(src_sd, KEY, direct_rdma=True)
    ctx.barrier()
    if reader:
        await ts.get_state_dict(KEY, user_state_dict=sh["dst"], direct_rdma=True)
    ctx.barrier()
    first_ms = (time.perf_counter() - t_first) * 1e3
    if reader:
        verify_flat(ctx, sh, "first sync")
    from torchstore_b200.state_dict_utils import _get_rdma_cache

    cl = await ts.client()
    dest_sync = _get_rdma_cache(cl).dests.get(KEY) if reader else None
    used_nccl = bool(args.allgather and all_readers and n > 1 and (dest_sync is None or dest_sync._plan is None))
    info = None
    if not used_nccl:
        info = pick_info(ctx, dest_sync if reader else None)

    async def step():
        await ts.put_state_dict(None, KEY, direct_rdma=True)
        if reader:
            await ts.get_state_dict(KEY, user_state_dict=sh["dst"], direct_rdma=True)

    kms = (lambda: dest_sync.last_pull_ms.get(ctx.local_rank)) if (reader and not used_nccl) else (lambda: None)
    timed = await timed_steps(ctx, step, kms, zero=(lambda: sh["dst_flat"].zero_()) if reader else None)
    if used_nccl:
        # NCCL runs on torch's stream: time it with wall clock + synchronize instead of copy-stream events
        ctx.barrier()
        t0 = time.perf_counter()
        for _ in range(args.steps):
            await step()
        torch.cuda.synchronize()
        timed["dev_ms"] = ctx.allmax((time.perf_counter() - t0) * 1e3)
        timed["kern_avg"] = timed["dev_ms"] / args.steps
    if reader:
        verify_flat(ctx, sh, "timed steps")
    ctx.barrier()
    if rank != 0:
        return None
    steps = args.steps
    value = sd_bytes * steps / (timed["dev_ms"] / 1e3) / 1e9
    readers = n if all_readers else 1
    remote_in = sd_bytes * (n - 1) // n  # bytes each reader ingests over NVLink
    if info is not None:
        roofline = roofline_for(n > 1, info, timed["kern_avg"])
    else:
        nvl = remote_in / (timed["kern_avg"] / 1e3) / 1e9
        roofline = {"bound": "nvlink", "achieved": nvl, "peak": NVLINK_NOMINAL_GBPS, "unit": "GB/s", "frac": nvl / NVLINK_NOMINAL_GBPS,
                    "traffic": None, "kernel": "ncclAllGather (library collective, 291 calls)", "kernel_ms_avg": timed["kern_avg"],
                    "algorithmic_bytes_per_launch": remote_in}
    return base_line(
        ctx, value, timed["dev_ms"] / steps,
        f"llama3-8b bf16 state_dict FSDP({n}) Shard(0) -> {'every rank' if all_readers else 'one reader (rank 0)'} reads the whole "
        f"state dict ({'NCCL all_gather route' if used_nccl else 'P2P pulls, one copy_rects launch per reader'}), "
        "ts.put_state_dict/get_state_dict(direct_rdma=True)",
        {"state_dict_bytes": sd_bytes, "readers": readers, "delivered_bytes_per_step": sd_bytes * readers,
         "nvlink_bytes_into_each_reader": remote_in, "route": "nccl_all_gather" if used_nccl else "p2p",
         "first_sync_ms_incl_registration_and_planning": first_ms, "wall_ms_per_step": timed["wall_ms"] / steps,
         "parity": "bit-exact torch.equal of every full tensor on every reader"},
        timed, roofline, None, None, remote_in / (timed["dev_ms"] / steps / 1e3) / 1e9 / NVLINK_NOMINAL_GBPS if n > 1 else 0.0)


# =================================================================================================
# config 5: store path put_batch / get_batch sweep
# =================================================================================================
async def cfg_store_sweep(ctx: Ctx):
    """Every rank puts flat bf16 keys into ITS volume (LocalRankStrategy: the HBM arena of its own GPU),
    reads them back in place (local D2D) and reads its neighbour's keys (P2P over NVLink).  Key size is
    swept 1 MiB .. 8 GiB at (up to) the Llama-3-70B per-GPU share of 17.6 GB per batch; small keys are
    capped at `max_keys` per batch and are latency-, not bandwidth-, limited (said in the result)."""
    torch, args = ctx.torch, ctx.args
    n, rank = ctx.world, ctx.rank
    import torchstore_b200 as ts_mod

    per_gpu = workloads.state_dict_bytes(workloads.llama_layout(workloads.LLAMA3_70B)) // 8  # 17.6 GB
    per_gpu = int(os.environ.get("TSB_SWEEP_BYTES", per_gpu))
    max_keys = int(os.environ.get("TSB_SWEEP_MAX_KEYS", "1024"))
    sizes = [1 << s for s in range(20, 34, 2)] + [8 << 30]  # 1 MiB, 4 MiB, ... 4 GiB, 8 GiB
    sizes = sorted(set(s for s in sizes if s <= per_gpu))
    os.environ.setdefault("TORCHSTORE_B200_SLAB_BYTES", str(max(4 << 30, per_gpu + (1 << 30))))
    ts = await init_store(ctx)
    def seeded(r):
        g = torch.Generator(device=ctx.dev)
        g.manual_seed(4242 + r)
        t = torch.empty(per_gpu // 2, dtype=torch.bfloat16, device=ctx.dev)
        t.view(torch.int16).random_(-32768, 32767, generator=g)  # arbitrary bit patterns
        return t

    src = seeded(rank)
    peer_src = seeded((rank + 1) % n) if n > 1 else None  # what the neighbour stored: expected result of a peer get
    dst = torch.zeros_like(src)
    rows = []
    launches0 = ctx.native.launch_count()
    sampler = ClockSampler(ctx.local_rank)
    if rank == 0:
        sampler.start()
    for key_bytes in sizes:
        nkeys = max(1, min(per_gpu // key_bytes, max_keys))
        total = nkeys * key_bytes
        el = key_bytes // 2
        mine = {f"sweep/r{rank}/k{i}": src[i * el:(i + 1) * el] for i in range(nkeys)}
        back = {f"sweep/r{rank}/k{i}": dst[i * el:(i + 1) * el] for i in range(nkeys)}
        peer = (rank + 1) % n
        theirs = {f"sweep/r{peer}/k{i}": dst[i * el:(i + 1) * el] for i in range(nkeys)}

        async def timed(coro_fn, reps):
            """median over reps of the slowest rank's wall time for one batch (barrier + synchronize around each)"""
            samples = []
            for _ in range(reps):
                ctx.barrier()
                t0 = time.perf_counter()
                await coro_fn()
                torch.cuda.synchronize()
                samples.append(ctx.allmax(time.perf_counter() - t0))
            return statistics.median(samples)

        reps = 5 if total <= (4 << 30) else 3
        await ts.put_batch(mine)  # first put allocates arena blocks; later puts overwrite in place
        if os.environ.get("TSB_BENCH_PROFILE") and rank == 0 and key_bytes == int(os.environ["TSB_BENCH_PROFILE"]):
            import cProfile
            import pstats

            prof = cProfile.Profile()
            prof.enable()
            await ts.put_batch(mine)
            await ts.get_batch(back)
            prof.disable()
            pstats.Stats(prof, stream=sys.stderr).sort_stats("cumulative").print_stats(45)
        t_put = await timed(lambda: ts.put_batch(mine), reps)
        dst.zero_()
        await ts.get_batch(back)  # warm-up: first get maps the volume's arena
        t_get = await timed(lambda: ts.get_batch(back), reps)
        ok = torch.equal(dst[: nkeys * el].view(torch.int16), src[: nkeys * el].view(torch.int16))
        t_peer = t_solo = None
        if n > 1:
            dst.zero_()
            await ts.get_batch(theirs)  # warm-up: cudaIpcOpenMemHandle of the peer's arena slab
            t_peer = await timed(lambda: ts.get_batch(theirs), reps)
            ok = ok and torch.equal(dst[: nkeys * el].view(torch.int16), peer_src[: nkeys * el].view(torch.int16))
            # the same get with ONE reader on the box (rank 0 pulls from rank 1's volume, nobody else moves
            # bytes): the unloaded NVLink rate of the store path, next to the all-ranks-at-once figure above
            solo = []
            for _ in range(reps):
                ctx.barrier()
                t0 = time.perf_counter()
                if rank == 0:
                    await ts.get_batch(theirs)
                    torch.cuda.synchronize()
                solo.append(ctx.allmax(time.perf_counter() - t0 if rank == 0 else 0.0))
            t_solo = statistics.median(solo)
        rows.append({"key_bytes": key_bytes, "keys_per_batch": nkeys, "batch_bytes_per_gpu": total,
                     "put_GBps_per_gpu": total / t_put / 1e9, "get_local_GBps_per_gpu": total / t_get / 1e9,
                     "get_peer_GBps_per_gpu": (total / t_peer / 1e9) if t_peer else None,
                     "get_peer_single_reader_GBps": (total / t_solo / 1e9) if t_solo else None,
                     "put_us_per_key": t_put / nkeys * 1e6, "get_us_per_key": t_get / nkeys * 1e6, "parity": bool(ok)})
        if not ok:
            raise SystemExit(f"[rank {rank}] PARITY FAILURE in store sweep at key size {key_bytes}")
        ctx.phase(f"sweep {key_bytes >> 20} MiB x {nkeys}: put {rows[-1]['put_GBps_per_gpu']:.0f} get {rows[-1]['get_local_GBps_per_gpu']:.0f} "
                  f"peer {rows[-1]['get_peer_GBps_per_gpu']} GB/s per GPU")
        ctx.barrier()
        await ts.delete_batch(list(mine))
        ctx.barrier()
    clocks = sampler.stop() if rank == 0 else None
    launches = int(ctx.allsum(ctx.native.launch_count() - launches0))
    if rank != 0:
        return None
    peaks, peak_src = load_peaks()
    best = max(rows, key=lambda r: r["put_GBps_per_gpu"])
    timed_stub = {"clocks": clocks, "launches": launches}
    roofline = {"bound": "hbm", "achieved": 2 * best["put_GBps_per_gpu"], "peak": peaks["hbm_gbs"], "unit": "GB/s",
                "frac": 2 * best["put_GBps_per_gpu"] / peaks["hbm_gbs"], "traffic": None, "peak_source": peak_src,
                "kernel": "copy_rects_kernel (one-shot plans of the store path)", "note": "put = local D2D: 2 bytes of HBM traffic per payload byte; "
                "wall clock through ts.put_batch incl. RPC handshake"}
    line = base_line(ctx, best["put_GBps_per_gpu"] * n, None,
                     f"store path ts.put_batch/get_batch of flat bf16 keys, {per_gpu} B per GPU per batch (Llama-3-70B / 8), key size sweep",
                     {"sweep": rows, "max_keys_per_batch": max_keys, "value_is": "aggregate put GB/s at the best key size"},
                     timed_stub, roofline, None, None, 0.0, scaling="weak")
    line["metric"] = "store put_batch GB/s (batch bytes / wall s)"
    return line


def run_config1(args):
    """BASELINE config #1: single-process ts.put / ts.get of a 1 MiB fp32 tensor via LocalRankStrategy
    over the host tier (POSIX shm + tsb_host_copy_rects).  Plumbing, no GPU: runs on any box."""
    import torch

    import torchstore_b200 as ts

    os.environ.pop("RANK", None)
    os.environ["LOCAL_RANK"] = "0"
    t = torch.arange(512 * 512, dtype=torch.float32).reshape(512, 512)
    dest = torch.zeros(512, 512)
    put_ms, get_ms = [], []

    async def main():
        await ts.initialize(num_storage_volumes=1, strategy=ts.LocalRankStrategy(ts.TransportType.SharedMemory))
        try:
            for i in range(args.warmup + args.steps):
                t.add_(1.0)
                t0 = time.perf_counter()
                await ts.put("w", t)
                t1 = time.perf_counter()
                out = await ts.get("w", dest)
                t2 = time.perf_counter()
                if out is not dest or not torch.equal(dest, t):
                    raise SystemExit("PARITY FAILURE in config 1")
                if i >= args.warmup:
                    put_ms.append((t1 - t0) * 1e3)
                    get_ms.append((t2 - t1) * 1e3)
        finally:
            await ts.shutdown()

    asyncio.run(main())
    nbytes = t.numel() * 4
    step_ms = statistics.median(put_ms) + statistics.median(get_ms)
    emit({
        "metric": "put+get GB/s of a 1 MiB fp32 tensor (host tier, plumbing)", "value": 2 * nbytes / (step_ms / 1e3) / 1e9,
        "unit": "GB/s", "n_gpus": 0, "steps": args.steps, "warmup": args.warmup, "ms_per_step": step_ms,
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": "single-process ts.put/ts.get of a [512,512] fp32 tensor via LocalRankStrategy, "
                               "TransportType.SharedMemory (POSIX shm host tier), no GPU", "bench_config": "1", "bytes": nbytes,
                   "put_ms_median": statistics.median(put_ms), "get_ms_median": statistics.median(get_ms),
                   "cores": os.cpu_count(), "parity": "bit-exact, in-place get returns the caller's tensor"},
        "gpu_launches": 0, "e2e": None, "roofline": None, "cpu_baseline": None,
    })


CONFIGS = {
    "4": cfg_headline,
    "4p": cfg_disjoint,
    "2": cfg_flat2,
    "3a": lambda ctx: cfg_replicated(ctx, all_readers=False),
    "3b": lambda ctx: cfg_replicated(ctx, all_readers=True),
    "5": cfg_store_sweep,
}


def run_ours(args):
    ctx = Ctx(args)
    import torchstore_b200 as ts

    async def main():
        return await CONFIGS[args.config](ctx)

    out = asyncio.run(main())
    ctx.done()
    if ctx.rank == 0 and out is not None:
        emit(out)

    async def fin():
        await ts.shutdown()

    try:
        asyncio.run(fin())
    except Exception as e:  # noqa: BLE001
        print(f"[rank {ctx.rank}] shutdown: {e}", file=sys.stderr)
    ctx.dist.barrier(device_ids=[ctx.local_rank])
    ctx.dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", choices=["ours", "reference"], default="ours")
    ap.add_argument("--config", choices=sorted(CONFIGS) + ["1"], default="4",
                    help="BASELINE.json config to run (default 4 = the headline FSDP(N)->TP(N) sync)")
    ap.add_argument("--allgather", action="store_true", help="config 3b: route through NCCL all_gather instead of P2P pulls")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--profiler-range", action="store_true",
                    help="cudaProfilerStart/Stop around the timed steps (for ncu --profile-from-start off)")
    ap.add_argument("--no-e2e", action="store_true", help="skip the host-input leg (profiling runs)")
    ap.add_argument("--dump-outputs", metavar="DIR",
                    help="config 4: after the timed steps, write the destination state dict of the last step as DIR/<name>.npy "
                         "(float32; tensors over their share of 64 MiB in all are a fixed seeded sample of elements)")
    args = ap.parse_args()
    if args.dump_outputs and (args.impl != "ours" or args.config != "4"):
        ap.error("--dump-outputs applies to the default config 4 of --impl ours")
    args.warmup = max(args.warmup, 3) if args.impl == "ours" else args.warmup
    capture_stdout()
    if args.impl == "reference":
        run_reference(args)
    elif args.config == "1":
        run_config1(args)
    else:
        run_ours(args)


if __name__ == "__main__":
    main()

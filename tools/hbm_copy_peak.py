"""Device-to-device copy rate of one GPU: the HBM roofline bench.py uses (HBM_COPY_MEASURED_GBPS).

    python tools/hbm_copy_peak.py

torch copy_ of a 4 GiB buffer, timed with CUDA events over 5 windows of 20 copies after 3 warm-up
copies; rate = read + write bytes over time.  Prints one JSON line with the GPU's name, power limit and
maximum SM clock, which belong beside the number.
"""

import json
import statistics
import subprocess

import torch


def main():
    n = 4 << 30
    a = torch.empty(n, dtype=torch.uint8, device="cuda")
    b = torch.empty_like(a)
    a.random_(0, 255)
    for _ in range(3):
        b.copy_(a)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps, rates = 20, []
    for _ in range(5):
        torch.cuda.synchronize()
        e0.record()
        for _ in range(reps):
            b.copy_(a)
        e1.record()
        e1.synchronize()
        rates.append(2 * n * reps / (e0.elapsed_time(e1) / 1e3) / 1e9)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                          "-i", str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"copy_GBps_read_plus_write_median": statistics.median(rates), "windows": rates, "bytes": n, "gpu": gpu}))


if __name__ == "__main__":
    main()

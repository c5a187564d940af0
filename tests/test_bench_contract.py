"""The JSON line bench.py prints is a contract with its readers: every required key must be there for the
HBM-bound (N=1) and the NVLink-bound (N>1) form, and no figure that was not measured may appear as a number."""

import importlib
import json
import os
import sys
import types

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bench():
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    return importlib.import_module("bench")


INFO = {"num_rects": 1194, "num_tiles": 22665, "payload_bytes": 2008031232, "src_bytes": 2008031232,
        "remote_src_bytes": 528948224, "num_link_tiles": 143815, "link_bytes": 528948224, "grid": 396, "block": 288,
        "tile_bytes": 65536, "num_vector_rects": 1194, "link_tile_bytes": 4096, "link_stages": 6}
REQUIRED = ["metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
            "dtype", "data", "config", "clocks", "e2e", "gpu_launches", "roofline", "cpu_baseline"]


def test_roofline_blocks_have_the_contract_keys_and_state_what_was_measured():
    b = _bench()
    hbm = b.roofline_for(False, dict(INFO, remote_src_bytes=0), 4.7)
    nvl = b.roofline_for(True, INFO, 0.81)
    for r in (hbm, nvl):
        for k in ("bound", "achieved", "peak", "unit", "frac", "traffic"):
            assert k in r
        assert abs(r["frac"] - r["achieved"] / r["peak"]) < 1e-12
        # hardware byte counters are not available: the traffic figures are null and say so
        assert r["traffic"] is None and r["traffic_source"] == "not measured"
    assert hbm["bound"] == "hbm" and nvl["bound"] == "nvlink" and nvl["nvlink_traffic"] is None
    assert hbm["achieved"] == pytest.approx((INFO["src_bytes"] + INFO["payload_bytes"]) / 4.7e-3 / 1e9, rel=1e-12)
    assert nvl["achieved"] == pytest.approx(INFO["remote_src_bytes"] / 0.81e-3 / 1e9, rel=1e-12)
    # each peak names where it comes from: the HBM copy peak was measured, the NVLink rate is nominal
    assert "measured" in hbm["peak_source"] and "H100" in hbm["peak_source"]
    assert nvl["peak"] == b.NVLINK_NOMINAL_GBPS and "nominal" in nvl["peak_source"]
    assert nvl["hbm"]["algorithmic_bytes_per_launch_incl_serving_peers"] == 2 * INFO["payload_bytes"]


def test_base_line_carries_every_contract_key():
    b = _bench()
    ctx = types.SimpleNamespace(world=8, args=types.SimpleNamespace(steps=30, warmup=3, config="4"), numa={"bound": True})
    timed = {"clocks": {"sm_mhz": 1965.0, "sm_max_mhz": 1965.0, "reasons": []}, "launches": 240}
    line = b.base_line(ctx, 18000.0, 0.85, "workload", {"state_dict_bytes": 16060522496}, timed,
                       b.roofline_for(True, INFO, 0.81),
                       {"value": 414.0, "unit": "GB/s", "h2d_bytes_per_step": 16060522496, "d2h_bytes_per_step": 1}, None, 0.7)
    for k in REQUIRED:
        assert k in line, k
    assert line["config"]["workload"] == "workload" and "model" not in line["config"]
    assert line["higher_is_better"] is True and line["n_gpus"] == 8 and line["gpu_launches"] == 240
    json.dumps(line)  # serialisable

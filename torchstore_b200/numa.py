"""NUMA placement of host staging memory.

On an 8-GPU box the GPUs hang off two CPU sockets; a pinned host buffer that lives on the other
socket's DRAM lowers the H2D rate of a rank.
The reference pins its shm segments with ``cudaHostRegister`` wherever the kernel happened to
place them (transport/shared_memory.py:55-96); here the staging buffer of a rank is first-touched by
a thread bound to the cores of the GPU's own NUMA node and only then page-locked.

Everything is read from sysfs; on boxes without that information the helpers are no-ops.
"""

from __future__ import annotations

import logging
import os

import torch

logger = logging.getLogger(__name__)


def _parse_cpulist(text: str) -> list[int]:
    cpus: list[int] = []
    for part in text.strip().split(","):
        if not part:
            continue
        if "-" in part:
            a, b = part.split("-")
            cpus.extend(range(int(a), int(b) + 1))
        else:
            cpus.append(int(part))
    return cpus


def gpu_pci_address(device: int) -> str | None:
    """'0000:1b:00.0' style sysfs name of a CUDA device."""
    try:
        props = torch.cuda.get_device_properties(device)
        return f"{props.pci_domain_id:04x}:{props.pci_bus_id:02x}:{props.pci_device_id:02x}.0"
    except Exception:
        pass
    try:
        import pynvml

        pynvml.nvmlInit()
        visible = os.environ.get("CUDA_VISIBLE_DEVICES")
        index = int(visible.split(",")[device]) if visible else device
        info = pynvml.nvmlDeviceGetPciInfo(pynvml.nvmlDeviceGetHandleByIndex(index))
        bus = info.busId.decode() if isinstance(info.busId, bytes) else info.busId
        return bus.lower()[-12:]
    except Exception:
        return None


def gpu_numa_node(device: int) -> int | None:
    addr = gpu_pci_address(device)
    if addr is None:
        return None
    try:
        with open(f"/sys/bus/pci/devices/{addr}/numa_node") as f:
            node = int(f.read().strip())
        return node if node >= 0 else None
    except (OSError, ValueError):
        return None


def node_cpus(node: int) -> list[int]:
    try:
        with open(f"/sys/devices/system/node/node{node}/cpulist") as f:
            return _parse_cpulist(f.read())
    except OSError:
        return []


def bind_to_gpu_numa(device: int) -> dict:
    """Restrict the calling thread (and threads it creates later) to the cores of the GPU's NUMA
    node, so that host memory it first-touches lands in that node's DRAM.  Returns what was done."""
    node = gpu_numa_node(device)
    if node is None:
        return {"bound": False, "reason": "no NUMA information for the GPU"}
    cpus = set(node_cpus(node))
    try:
        allowed = os.sched_getaffinity(0)
    except AttributeError:
        return {"bound": False, "reason": "sched_getaffinity unavailable"}
    target = cpus & allowed
    if not target:
        return {"bound": False, "node": node, "reason": "no allowed core on the GPU's node"}
    try:
        os.sched_setaffinity(0, target)
    except OSError as e:
        return {"bound": False, "node": node, "reason": str(e)}
    return {"bound": True, "node": node, "cpus": len(target)}


def pinned_like(nbytes: int, dtype: torch.dtype = torch.uint8) -> torch.Tensor:
    """Page-locked host tensor of ``nbytes`` bytes whose pages were first touched by the calling
    thread (bind it with :func:`bind_to_gpu_numa` first).  Registered through the C-ABI
    (tsb_host_register), so async H2D/D2H copies from it run at full PCIe rate."""
    from torchstore_b200 import _native

    assert nbytes % dtype.itemsize == 0
    import ctypes

    t = torch.empty(nbytes // dtype.itemsize, dtype=dtype)
    # first touch happens HERE, on this thread (not on torch's intra-op pool, whose threads may have
    # been created before the binding)
    ctypes.memset(t.data_ptr(), 0, nbytes)
    _native.host_register(t.data_ptr(), nbytes)
    return t

"""Host-side placement for the host-buffer entry point (``LiftSplat.lift_from_host``): one process per GPU, each bound to the
CPU cores of its GPU's NUMA node BEFORE it allocates pinned memory, so the 36 MB up / 82 MB down per 8-frame step cross PCIe
into local DRAM instead of the inter-socket link (an 8-GPU HGX box has GPUs 0-3 on socket 0 and 4-7 on socket 1).

Linux only (sysfs); everything degrades to a no-op with a reason string when the information is not available.
"""
from __future__ import annotations

import os
from typing import List, Optional, Tuple

import torch


def _parse_cpulist(text: str) -> List[int]:
    cpus: List[int] = []
    for part in text.strip().split(","):
        if not part:
            continue
        if "-" in part:
            lo, hi = part.split("-")
            cpus.extend(range(int(lo), int(hi) + 1))
        else:
            cpus.append(int(part))
    return cpus


def gpu_numa_node(device_index: int) -> Optional[int]:
    """NUMA node of a CUDA device from sysfs (``/sys/bus/pci/devices/<domain:bus:dev.fn>/numa_node``), or None."""
    try:
        p = torch.cuda.get_device_properties(device_index)
        bdf = f"{p.pci_domain_id:04x}:{p.pci_bus_id:02x}:{p.pci_device_id:02x}.0"
        with open(f"/sys/bus/pci/devices/{bdf}/numa_node") as fh:
            node = int(fh.read().strip())
        return node if node >= 0 else None
    except (OSError, ValueError, AttributeError, RuntimeError):
        return None


def node_cpus(node: int) -> List[int]:
    try:
        with open(f"/sys/devices/system/node/node{node}/cpulist") as fh:
            return _parse_cpulist(fh.read())
    except OSError:
        return []


def bind_to_gpu_numa(device_index: int, local_rank: int = 0, ranks_on_node: int = 1) -> Tuple[Optional[int], int, str]:
    """Restricts this process to the cores of the GPU's NUMA node (a disjoint slice per rank when several ranks share a node),
    so that memory pinned afterwards is first-touched there.  Returns (node, cores bound, note)."""
    node = gpu_numa_node(device_index)
    if node is None:
        return None, 0, "numa node of the GPU unknown (no sysfs entry)"
    cpus = node_cpus(node)
    try:
        allowed = sorted(set(cpus) & set(os.sched_getaffinity(0)))
    except (AttributeError, OSError):
        return node, 0, "sched_getaffinity unavailable"
    if not allowed:
        return node, 0, "no allowed cores on the GPU's node"
    if ranks_on_node > 1:
        per = max(1, len(allowed) // ranks_on_node)
        k = local_rank % ranks_on_node
        mine = allowed[k * per:(k + 1) * per] or allowed
    else:
        mine = allowed
    try:
        os.sched_setaffinity(0, mine)
    except OSError as e:
        return node, 0, f"sched_setaffinity failed: {e}"
    return node, len(mine), "bound"

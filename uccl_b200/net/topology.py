"""GPU <-> NIC matching for rail-aligned multi-node jobs.

Each local rank should drive the NIC that hangs off the same PCIe switch as its GPU (on an H100 HGX board:
one ConnectX per GPU pair / GPU), so that staging traffic never crosses the CPU interconnect and every
rail uses its own NIC.  The reference does this in its RDMA bring-up by comparing sysfs PCI paths
(collective/rdma/util_rdma.*: GPU <-> NIC distance matrix).  Here it is a small pure function over the
same sysfs data, so it is testable without the hardware.
"""
from __future__ import annotations

import os
from typing import Callable, List, Optional, Sequence, Tuple

from . import list_interfaces


def pci_distance(path_a: str, path_b: str) -> int:
    """Hops between two devices in the PCIe tree given their resolved sysfs paths
    (``/sys/devices/pci0000:17/0000:17:01.0/0000:18:00.0/...``): edges up to the deepest common ancestor and
    down again.  Devices under different root complexes get a large constant on top (they talk through the
    CPU interconnect)."""
    a = [p for p in path_a.split("/") if p]
    b = [p for p in path_b.split("/") if p]
    common = 0
    for x, y in zip(a, b):
        if x != y:
            break
        common += 1
    dist = (len(a) - common) + (len(b) - common)
    roots = [next((p for p in parts if p.startswith("pci")), None) for parts in (a, b)]
    if roots[0] != roots[1]:
        dist += 100
    return dist


def _sysfs_nic_path(ifname: str) -> Optional[str]:
    p = f"/sys/class/net/{ifname}/device"
    return os.path.realpath(p) if os.path.exists(p) else None


def _sysfs_gpu_path(gpu_index: int) -> Optional[str]:
    try:
        import torch

        bus = torch.cuda.get_device_properties(gpu_index).pci_bus_id  # "0000:1B:00.0" (recent torch)
    except Exception:  # noqa: BLE001
        return None
    if isinstance(bus, int):
        return None
    p = f"/sys/bus/pci/devices/{str(bus).lower()}"
    return os.path.realpath(p) if os.path.exists(p) else None


def rank_nics(gpu_path: Optional[str], nics: Sequence[Tuple[str, str, Optional[str]]]) -> List[Tuple[int, str, str]]:
    """Sort ``(name, ip, sysfs_path)`` NICs by PCIe distance to the GPU (unknown paths last, stable)."""
    scored = []
    for order, (name, ip, path) in enumerate(nics):
        d = pci_distance(gpu_path, path) if (gpu_path and path) else 10_000 + order
        scored.append((d, name, ip))
    return sorted(scored, key=lambda t: t[0])


def nic_for_gpu(gpu_index: Optional[int] = None, local_rank: int = 0,
                interfaces: Optional[Sequence[Tuple[str, str]]] = None,
                nic_path: Callable[[str], Optional[str]] = _sysfs_nic_path,
                gpu_path: Callable[[int], Optional[str]] = _sysfs_gpu_path) -> Tuple[str, str]:
    """(interface name, ipv4) this rank should bind its transport engine to.

    With PCI information: the closest NIC; several equally close NICs (or no PCI information at all) are
    shared round-robin by ``local_rank``, which is what keeps rails disjoint on symmetric boards."""
    ifs = list(interfaces if interfaces is not None else list_interfaces())
    if not ifs:
        return ("lo", "127.0.0.1")
    nics = [(n, ip, nic_path(n)) for n, ip in ifs]
    gp = gpu_path(gpu_index) if gpu_index is not None else None
    ranked = rank_nics(gp, nics)
    best = ranked[0][0]
    ties = [r for r in ranked if r[0] == best] if best < 10_000 else ranked
    _, name, ip = ties[local_rank % len(ties)]
    return (name, ip)

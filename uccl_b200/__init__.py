"""uccl_b200 -- a Hopper-native (sm_90a, NVLink 4 / NVSwitch) GPU communication library
with the capabilities of uccl-project/uccl:

* ``uccl_b200.collective``  NCCL-style collectives (hand-written P2P / NVLS kernels over a
  symmetric heap) + torch ProcessGroup glue + DDP hooks
* ``uccl_b200.ep``          DeepEP-compatible expert-parallel dispatch / combine
* ``uccl_b200.p2p``         NIXL-style initiator/target transfer engine (KV-cache moves)
* ``uccl_b200.ukernel``     launch-free collectives: persistent worker kernel + CCL planner
* ``uccl_b200.net``         scale-out: multipath reliable datagram transport between boxes, NCCL net
  plugin, ``parallel.MultiNodeCommunicator`` (NVLink inside a box, one rail per NIC between boxes)
* ``uccl_b200.models``      ResNet (DDP example), expert-parallel MoE layer (inference + training)

Everything also runs on a CPU-only machine through reference backends (host communicators,
``ep.Buffer(comm=<host comm>)``, ``p2p.Endpoint(-1)``, ``ukernel.Worker(device=-1)``).

Reference entry points mirrored: ``uccl/__init__.py:12-54`` (version + library path helpers).
"""
from __future__ import annotations

import os

__version__ = "0.1.0"

from . import _native  # noqa: E402


def lib_dir() -> str:
    return os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib")


def nccl_shim_path() -> str:
    """Absolute path of the NCCL-API drop-in (``libuccl_b200_nccl.so``).

    On one NVSwitch node no byte ever reaches a net plugin, so the intra-node drop-in is the NCCL *API*
    itself (``LD_PRELOAD``); the net plugin for traffic between nodes is :func:`nccl_plugin_path`."""
    return os.path.join(lib_dir(), "libuccl_b200_nccl.so")


def nccl_plugin_path() -> str:
    """Absolute path of the NCCL *network* plugin (``libnccl-net-uccl_b200.so``, ``ncclNet_v8``): what
    ``NCCL_NET_PLUGIN`` should point at for inter-node traffic (reference: ``uccl.nccl_plugin_path()``)."""
    return os.path.join(lib_dir(), "libnccl-net-uccl_b200.so")


def build(force: bool = False):
    from . import _build

    return _build.build(force=force)


from .parallel.comm import Communicator  # noqa: E402,F401

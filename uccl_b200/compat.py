"""Run code written against the reference's ``uccl`` package unchanged:

    import uccl_b200.compat; uccl_b200.compat.install()      # once, before the first `import uccl`
    from uccl import p2p, collective                         # -> uccl_b200.p2p / uccl_b200.collective
    from uccl.ep import Buffer                               # -> uccl_b200.ep

``install()`` registers module aliases in ``sys.modules`` (``uccl``, ``uccl.p2p``, ``uccl.collective``, ``uccl.utils``,
``uccl.ep``)
and refuses to shadow a real ``uccl`` distribution that is already imported.  The reference's package root offers
``nccl_plugin_path`` / ``rccl_plugin_path`` / ``efa_plugin_path`` / ``efa_nccl_path`` (uccl/__init__.py:12-54): the first
exists here, the other three name libraries of other hardware and raise.
"""
from __future__ import annotations

import sys
import types


def install(name: str = "uccl") -> types.ModuleType:
    import uccl_b200
    import uccl_b200.collective
    import uccl_b200.ep
    import uccl_b200.p2p
    import uccl_b200.p2p.utils

    cur = sys.modules.get(name)
    if cur is not None and getattr(cur, "__uccl_b200_alias__", False):
        return cur
    if cur is not None:
        raise RuntimeError(f"a different '{name}' package is already imported ({getattr(cur, '__file__', '?')})")
    m = types.ModuleType(name, "alias of uccl_b200 (installed by uccl_b200.compat.install)")
    m.__uccl_b200_alias__ = True
    m.__version__ = uccl_b200.__version__
    m.__path__ = []  # a package: `import uccl.p2p` consults sys.modules first
    m.p2p, m.collective, m.ep = uccl_b200.p2p, uccl_b200.collective, uccl_b200.ep
    m.utils = uccl_b200.p2p.utils  # the reference ships p2p/utils.py as uccl/utils.py (build_inner.sh:183)
    m.has_efa = lambda: False  # uccl/__init__.py:12-20: an NVLink box has no EFA devices to prefer
    m.is_efa = False
    m.nccl_plugin_path = uccl_b200.nccl_plugin_path
    m.nccl_shim_path = uccl_b200.nccl_shim_path

    def _other_hardware(what):
        def f():
            raise NotImplementedError(f"uccl_b200 is an sm_90a / NVLink library: there is no {what}")

        return f

    m.rccl_plugin_path = _other_hardware("RCCL plugin")
    m.efa_plugin_path = _other_hardware("EFA plugin")
    m.efa_nccl_path = _other_hardware("EFA build of NCCL")
    sys.modules[name] = m
    for sub in ("p2p", "collective", "ep", "utils"):
        sys.modules[f"{name}.{sub}"] = getattr(m, sub)
    return m


def install_ukernel() -> None:
    """Aliases for the reference's experimental ukernel packages: ``ukernel_ccl`` (ProcessGroup + functional API,
    experimental/ukernel/py/ukernel_ccl) -> ``uccl_b200.ukernel`` and ``ukernel_p2p`` (rank-addressed Communicator,
    experimental/ukernel/py/ukernel_p2p) -> ``uccl_b200.ukernel.p2p``."""
    import uccl_b200.ukernel
    import uccl_b200.ukernel.p2p

    for name, mod in (("ukernel_ccl", uccl_b200.ukernel), ("ukernel_p2p", uccl_b200.ukernel.p2p)):
        cur = sys.modules.get(name)
        if cur is not None and cur is not mod:
            raise RuntimeError(f"a different '{name}' module is already imported ({getattr(cur, '__file__', '?')})")
        sys.modules[name] = mod


def uninstall(name: str = "uccl") -> None:
    for extra, target in (("ukernel_ccl", "uccl_b200.ukernel"), ("ukernel_p2p", "uccl_b200.ukernel.p2p")):
        if sys.modules.get(extra) is sys.modules.get(target) and extra in sys.modules:
            sys.modules.pop(extra)
    cur = sys.modules.get(name)
    if cur is not None and getattr(cur, "__uccl_b200_alias__", False):
        for k in [name] + [f"{name}.{s}" for s in ("p2p", "collective", "ep", "utils")]:
            sys.modules.pop(k, None)

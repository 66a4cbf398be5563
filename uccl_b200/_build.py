"""In-tree native build: nvcc (sm_90a) for the kernels, host compiler for the runtime.

Everything is compiled with ``-gencode arch=compute_90a,code=sm_90a -lineinfo`` and linked
into ``uccl_b200/_C.<abi>.so`` (pybind11 module) next to this file, so the shared object
travels with the repo snapshot to the GPU box.  Incremental: an object is rebuilt when its
source or any header under csrc/ is newer.

Reference counterpart: build.sh / build_inner.sh / ep/setup.py (docker + setuptools); here a
single dependency-free script, because the target is exactly one architecture.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

ROOT = Path(__file__).resolve().parent
CSRC = ROOT / "csrc"
BUILD = ROOT.parent / "build" / "obj"

ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC = os.environ.get("NVCC", shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc")


def _ext_suffix() -> str:
    return sysconfig.get_config_var("EXT_SUFFIX") or ".so"


def module_path() -> Path:
    return ROOT / ("_C" + _ext_suffix())


def nccl_shim_path() -> Path:
    return ROOT / "lib" / "libuccl_b200_nccl.so"


def nccl_net_plugin_path() -> Path:
    """NCCL network plugin (inter-node transport): ``NCCL_NET_PLUGIN=uccl_b200`` resolves to this name."""
    return ROOT / "lib" / "libnccl-net-uccl_b200.so"


def _sources():
    cu = sorted(CSRC.glob("kernels/*.cu")) + sorted(CSRC.glob("ep/*.cu")) + sorted(CSRC.glob("p2p/*.cu"))
    cu += sorted(CSRC.glob("ukernel/*.cu"))
    cc = (
        sorted(CSRC.glob("fabric/*.cc"))
        + sorted(CSRC.glob("coll/*.cc"))
        + sorted(CSRC.glob("ep/*.cc"))
        + sorted(CSRC.glob("p2p/*.cc"))
        + sorted(CSRC.glob("common/*.cc"))
        + sorted(CSRC.glob("ukernel/*.cc"))
        + sorted(CSRC.glob("net/*.cc"))
    )
    bind = sorted(CSRC.glob("bind/*.cc"))
    return cu, cc, bind


def _newest_header() -> float:
    t = 0.0
    for pat in ("**/*.h", "**/*.cuh", "**/*.hpp"):
        for h in CSRC.glob(pat):
            t = max(t, h.stat().st_mtime)
    return t


def _includes():
    import pybind11

    return [
        "-I" + str(CSRC),
        "-I" + pybind11.get_include(),
        "-I" + sysconfig.get_paths()["include"],
        "-I/usr/local/cuda/include",
        "-I/usr/include",
    ]


def _compile_one(src: Path, obj: Path, verbose: bool) -> None:
    common = ["-std=c++17", "-O3", "-lineinfo", "-Xcompiler", "-fPIC,-fvisibility=hidden,-Wall,-Wno-unused-function"]
    cmd = [NVCC] + ARCH_FLAGS + common + _includes()
    if src.suffix == ".cu":
        cmd += ["-Xptxas", "-v"] if verbose else []
    cmd += ["-c", str(src), "-o", str(obj)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError(f"compile failed: {src}")
    if verbose and r.stderr:
        (obj.with_suffix(".ptxas.txt")).write_text(r.stderr)


def build(force: bool = False, verbose: bool = False, jobs: int | None = None) -> Path:
    """Compile every CUDA/C++ source for sm_90a and link the python module. Returns its path."""
    if not Path(NVCC).exists():
        raise RuntimeError(f"nvcc not found at {NVCC}")
    BUILD.mkdir(parents=True, exist_ok=True)
    cu, cc, bind = _sources()
    hdr_t = _newest_header()
    this_t = Path(__file__).stat().st_mtime
    todo, objs = [], []
    for src in cu + cc + bind:
        obj = BUILD / (src.parent.name + "_" + src.stem + ".o")
        objs.append(obj)
        if force or not obj.exists() or obj.stat().st_mtime < max(src.stat().st_mtime, hdr_t, this_t):
            todo.append((src, obj))
    jobs = jobs or max(1, (os.cpu_count() or 4))
    if todo:
        with ThreadPoolExecutor(max_workers=jobs) as ex:
            list(ex.map(lambda so: _compile_one(so[0], so[1], verbose), todo))
    out = module_path()
    shim_objs = [o for o in objs if o.name == "coll_nccl_shim.o"]
    plugin_objs = [o for o in objs if o.name == "net_nccl_net_plugin.o"]
    bind_objs = [o for o in objs if o.name.startswith("bind_") or "_bind_" in o.name]
    core_objs = [o for o in objs if o not in shim_objs and o not in bind_objs and o not in plugin_objs]

    def link(target: Path, these):
        target.parent.mkdir(parents=True, exist_ok=True)
        cmd = [NVCC] + ARCH_FLAGS + ["-shared", "-o", str(target)] + [str(o) for o in these] + ["-lrt", "-lpthread", "-ldl"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError(f"link failed: {target}")

    if todo or not out.exists():
        link(out, core_objs + bind_objs)
    shim = nccl_shim_path()
    if shim_objs and (todo or not shim.exists()):
        # NCCL-API drop-in: same kernels/runtime, nccl.h symbols, no python
        link(shim, core_objs + shim_objs)
    plugin = nccl_net_plugin_path()
    if plugin_objs and (todo or not plugin.exists()):
        # NCCL net plugin: host-only code (sockets), no CUDA runtime dependency
        net_core = [o for o in core_objs if o.name == "net_net_engine.o"]
        cmd = ["g++", "-shared", "-o", str(plugin)] + [str(o) for o in plugin_objs + net_core] + ["-lpthread"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError(f"link failed: {plugin}")
    return out


def ensure_built() -> Path:
    out = module_path()
    if not out.exists():
        build()
    return out


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(p)

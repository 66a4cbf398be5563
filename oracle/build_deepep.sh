#!/bin/bash
# Builds the reference's vendored upstream DeepEP (thirdparty/DeepEP, sources untouched) for sm_90a with
# its own setup.py and installs it under oracle/_ref/deepep (git-ignored).
#
#   bash oracle/build_deepep.sh <checkout of uccl-project/uccl>
# Its setup.py enables NVSHMEM whenever the `nvidia.nvshmem` wheel is importable; the IBGDA headers that
# path needs (infiniband/mlx5dv.h) are absent here, so the wheel is hidden from find_spec to take the
# script's own DISABLE_NVSHMEM branch (intranode kernels only -- exactly what the EP=8 headline uses).
set -euo pipefail
ROOT="$(cd "$(dirname "$0")/.." && pwd)"
REF="${1:?usage: oracle/build_deepep.sh <checkout of uccl-project/uccl>}/thirdparty/DeepEP"
WORK="${TMPDIR:-/tmp}/deepep_build"
rm -rf "$WORK" && cp -r "$REF" "$WORK"
cd "$WORK"
python - <<'EOF'
import importlib.util, os, sys
_orig = importlib.util.find_spec
def _fs(name, *a, **k):
    if name == "nvidia.nvshmem":
        raise ModuleNotFoundError(name)
    return _orig(name, *a, **k)
importlib.util.find_spec = _fs
os.environ["TORCH_CUDA_ARCH_LIST"] = "9.0a"   # its setup.py keeps the aggressive PTX loads off by default
os.environ.setdefault("MAX_JOBS", "8")
sys.argv = ["setup.py", "build_ext", "--inplace"]
exec(compile(open("setup.py").read(), "setup.py", "exec"), {"__name__": "__main__", "__file__": "setup.py"})
EOF
# Its setup.py compiles with -rdc=true but only adds the device-link step on the NVSHMEM branch, so the
# module it links has an unresolved __cudaRegisterLinkedBinary_*; do the device link here (objects untouched).
T="$(echo build/temp.*/csrc)"
nvcc -dlink -Xcompiler -fPIC -Xnvlink -ignore-host-info -gencode=arch=compute_90a,code=sm_90a "$T"/kernels/intranode.o "$T"/kernels/layout.o \
  "$T"/kernels/runtime.o -o "$T"/dlink.o
TORCH_LIB="$(python -c 'import torch, os; print(os.path.join(os.path.dirname(torch.__file__), "lib"))')"
g++ -shared "$T"/deep_ep.o "$T"/kernels/intranode.o "$T"/kernels/layout.o "$T"/kernels/runtime.o "$T"/dlink.o \
  -L"$TORCH_LIB" -L/usr/local/cuda/lib64 -lc10 -ltorch -ltorch_cpu -ltorch_python -lcudart -lcudadevrt -lc10_cuda \
  -ltorch_cuda -o "$(ls deep_ep_cpp*.so)"
mkdir -p "$ROOT/oracle/_ref/deepep"
rm -rf "$ROOT/oracle/_ref/deepep/deep_ep"
cp -r deep_ep "$ROOT/oracle/_ref/deepep/"
cp deep_ep_cpp*.so "$ROOT/oracle/_ref/deepep/"
echo "installed: $ROOT/oracle/_ref/deepep"

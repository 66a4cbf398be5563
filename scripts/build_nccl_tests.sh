#!/bin/bash
# Builds the reference's vendored nccl-tests (thirdparty/nccl-tests, unmodified, its own Makefile) for sm_90a
# against the system NCCL headers into build/nccl-tests.  The same binaries are then run twice: as they are
# (system NCCL 2.27 = the baseline the reference's run_nccl_test.sh measures) and with the NCCL-API drop-in
# preloaded (scripts/run_nccl_tests.sh).  Reference: collective/rdma/run_nccl_test.sh:41-49,95-98,
# experimental/lite/scripts/run-nccl-tests.sh:36-60.
set -euo pipefail
ROOT="$(cd "$(dirname "$0")/.." && pwd)"
SRC="${1:?usage: scripts/build_nccl_tests.sh <checkout of uccl-project/uccl>}/thirdparty/nccl-tests"
mkdir -p "$ROOT/build/nccl-tests"
make -C "$SRC/src" -j"$(nproc)" BUILDDIR="$ROOT/build/nccl-tests" \
  NVCC_GENCODE="-gencode=arch=compute_90a,code=sm_90a" NCCL_HOME=/usr
ls "$ROOT"/build/nccl-tests/*_perf

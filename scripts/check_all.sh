#!/usr/bin/env bash
# Everything that can be checked without a GPU, in the order the CI runs it:
#   build for sm_90a -> CPU test-suite -> transport under ASan/UBSan and TSan -> GPU tests only collected.
# With --profiles the CPU-side scale-out measurements under profiles/ are regenerated as well.
set -euo pipefail
ROOT="$(cd "$(dirname "$0")/.." && pwd)"
cd "$ROOT"
python -c "import __graft_entry__ as g; g.build(); print('build: ok')"
python -m pytest tests -x -q -m "not gpu"
for san in address,undefined thread; do
  g++ -std=c++17 -O1 -g -fsanitize=$san -Iuccl_b200/csrc tests/cpp/net_engine_test.cc uccl_b200/csrc/net/net_engine.cc -o /tmp/net_san_$$ -lpthread
  ASAN_OPTIONS=detect_leaks=0 /tmp/net_san_$$ 3 swift 8 | tail -1
  rm -f /tmp/net_san_$$
done
# (the P2P engine stress and the ukernel planner run under TSan / ASan+UBSan from inside the pytest suite:
#  tests/test_host_p2p.py::test_engine_concurrency_stress_under_sanitizers, tests/test_ukernel.py::test_planner_cpp_unit_under_sanitizers)
for san in thread address; do bash scripts/sanitize_host.sh $san | tail -1; done
python -m pytest tests -m gpu --collect-only -q | tail -1
if [ "${1:-}" = "--profiles" ]; then ./scripts/run_scaleout_cpu.sh; fi
echo "check_all: ok"

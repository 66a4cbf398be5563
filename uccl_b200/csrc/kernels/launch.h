// Host-callable launchers of every kernel (implemented in the .cu translation units).
#pragma once
#include <cuda_runtime.h>

#include "types.h"

namespace ub {
// CUDA lazy module loading may need a context synchronisation when a kernel is launched for
// the first time; if another kernel of this process is spinning on a peer that has not been
// launched yet (single-process multi-rank worlds) that is a deadlock.  preload_all_kernels()
// walks every launcher in "preload mode" (cudaFuncGetAttributes instead of a launch) so all
// functions are resident before the first collective.
extern bool g_preload;
cudaError_t preload_all_kernels();
#define UB_LAUNCH(kern, grid, block, smem, st, ...)                         \
  do {                                                                     \
    auto _ub_k = kern;                                                     \
    if (::ub::g_preload) {                                                 \
      cudaFuncAttributes _ub_fa;                                           \
      cudaError_t _ub_e = cudaFuncGetAttributes(&_ub_fa, _ub_k);           \
      if (_ub_e != cudaSuccess) return _ub_e;                              \
    } else {                                                               \
      _ub_k<<<grid, block, smem, st>>>(__VA_ARGS__);                       \
    }                                                                      \
  } while (0)

// allreduce: algo ids = ArAlgo in allreduce_impl.cuh (same numbering as ArAlgoId in comm.h)
cudaError_t launch_allreduce_f(int algo, int dtype, int op, int out_dtype, const DevComm& c, const CollArgs& a,
                               int grid, int block, cudaStream_t st);
cudaError_t launch_allreduce_i(int algo, int dtype, int op, const DevComm& c, const CollArgs& a, int grid,
                               int block, cudaStream_t st);
cudaError_t launch_allreduce_x(int algo, int dtype, int op, const DevComm& c, const CollArgs& a, int grid,
                               int block, cudaStream_t st);
// all-reduce (sum) + residual add + RMSNorm [+ e4m3 cast] (allreduce_rmsnorm.cu): algo AR_ONESHOT_LL / AR_ONESHOT_MC
// launch the fused one-shot kernel (a = one-shot arguments with in = out = r.x), algo 0 the local epilogue on an
// already reduced r.x.  dtype kBF16 / kF16; fp8 = e4m3 output with per-128-channel scales.
cudaError_t launch_allreduce_rmsnorm(int algo, int dtype, bool fp8, const DevComm& c, const CollArgs& a,
                                     const RmsNormArgs& r, int grid, cudaStream_t st);
// LL reduce-scatter (sum) + residual add + RMSNorm [+ e4m3 cast] (allreduce_rmsnorm.cu): a = LL reduce-scatter
// arguments with in = the whole x and bytes = one rank's piece; r = this rank's shard (r.x = its piece of x, r.T = its
// rows).  Block size kRmsThreads; bytes % 16 == 0.
cudaError_t launch_reduce_scatter_rmsnorm(int dtype, bool fp8, const DevComm& c, const CollArgs& a,
                                          const RmsNormArgs& r, int grid, cudaStream_t st);
// allgather modes: 0 push P2P, 1 push multicast, 2 pull/staged, 3 LL packets, 4 LL packets via multicast
cudaError_t launch_allgather(int mode, const DevComm& c, const CollArgs& a, int grid, int block, cudaStream_t st);
cudaError_t launch_broadcast(int mode, const DevComm& c, const CollArgs& a, int grid, int block, cudaStream_t st);
// alltoall modes: 0 pull/staged, 1 push, 2 LL packets
cudaError_t launch_alltoall(int mode, const DevComm& c, const CollArgs& a, int grid, int block, cudaStream_t st);
cudaError_t launch_alltoallv(const DevComm& c, const CollArgs& a, const A2AvArgs& v, int grid, int block,
                             cudaStream_t st);
// which: 0 = reduce_scatter, 1 = reduce
cudaError_t launch_red_f(int which, int dtype, int op, bool nvls, const DevComm& c, const CollArgs& a, int grid,
                         int block, cudaStream_t st);
cudaError_t launch_red_i(int which, int dtype, int op, const DevComm& c, const CollArgs& a, int grid, int block,
                         cudaStream_t st);
// barrier-free LL ReduceScatter (ll_exchange.cuh); bytes per rank % 16 == 0
cudaError_t launch_rs_ll_f(int dtype, int op, const DevComm& c, const CollArgs& a, int grid, int block,
                           cudaStream_t st);
cudaError_t launch_rs_ll_i(int dtype, int op, const DevComm& c, const CollArgs& a, int grid, int block,
                           cudaStream_t st);
cudaError_t launch_sendrecv(const DevComm& c, const SendRecvArgs& a, cudaStream_t st);
cudaError_t launch_barrier(const DevComm& c, int domain, cudaStream_t st);
// out[b] = SM id CTA b ran on; every CTA holds its SM for hold_ns (probe.cu)
cudaError_t launch_smid_probe(int* out, int blocks, unsigned long long hold_ns, cudaStream_t st);
}  // namespace ub

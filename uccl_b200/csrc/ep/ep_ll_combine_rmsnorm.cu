// Low-latency (decode) EP combine fused with the residual add and RMSNorm that end a decode MoE layer, optionally
// quantised to e4m3 for the next layer's fp8 GEMM or dispatch:
//
//   routed       = bf16(0 + sum over k ascending of w[t,k] * expert row k, skipping unrouted entries)   (fp32)
//   combined     = routed, or bf16(routed + shared) with a shared-expert output
//   residual_out = bf16(combined + residual)
//   out          = bf16(residual_out * rsqrt(mean(residual_out^2) + eps) * weight)   [-> e4m3 + scales]
//
// routed is exactly what ep_ll_combine_kernel writes, and combined exactly torch's bf16 routed + shared, but neither
// is stored: the row stays in registers and goes straight into the row epilogue of rmsnorm_row.cuh, the one
// add_rmsnorm_kernel runs.  So the result is bitwise that of low_latency_combine, + shared and add_rmsnorm_kernel.
//
// Block protocol of ep_ll_combine_kernel (one 512-thread block per token, the same grid, the same sync calls), so it
// interleaves with LL dispatch and combine on one stream, in hooks and in CUDA graphs.  Only the FULL and RECV
// phases run here: the SEND half of a hook split is ep_ll_combine_kernel's, which only announces that this rank's
// expert outputs are in place.
//
// Row-owned: block b owns tokens b, b + grid, ...  Chunk i = warp * 32 + lane + j * 512 of ep_ll_combine_kernel is
// unit j * kRmsThreads + threadIdx.x of the epilogue, and H <= 8192 gives at most kLLUnits = 2 units per thread.  A
// token's residual, shared and first expert-row loads are issued before the first add; its send_pos / topk_weights
// entries were fetched while the previous token ran.
#include "../kernels/launch.h"
#include "../kernels/rmsnorm_row.cuh"
#include "ep_buffer.h"
#include "ep_common.cuh"

namespace ub {

namespace {

constexpr int kLLUnits = 2;  // 16-byte units per thread: H <= 8192 = 2 * kRmsThreads * 8

// Chunk i of a token's routed row in fp32: the expression of ep_ll_combine_kernel, in the same order (0, then
// w[k] * row k for k ascending; entries k < 9 from registers, v[k] loaded when rowp[k] && valid, the rest loaded
// here from lane k's send_pos / weight).  That kernel keeps its own copy of these lines: calling this helper from it
// changes its register allocation and spills.  All 32 lanes of the warp must call this with the same K.
__device__ __forceinline__ void ll_weighted_sum(float (&acc)[8], const uint4 (&v)[9], const char* const (&rowp)[9],
                                                const float (&wk)[9], bool valid, long long pos, float w, int K,
                                                const DevComm& c, uint64_t x_off, size_t row_bytes, uint32_t i) {
#pragma unroll
  for (int q = 0; q < 8; ++q) acc[q] = 0.f;
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    if (rowp[k] && valid) {
      float f[8];
      bf16x8_to_float(v[k], f);
#pragma unroll
      for (int q = 0; q < 8; ++q) acc[q] += wk[k] * f[q];
    }
  }
  for (int k = 9; k < K; ++k) {
    const long long pk = __shfl_sync(0xffffffffu, pos, k);
    const float wkk = __shfl_sync(0xffffffffu, w, k);
    if (pk >= 0 && valid) {
      float f[8];
      bf16x8_to_float(ld_nc_v4(c.heap[(int)(pk >> 32)] + x_off + (size_t)(pk & 0xffffffffll) * row_bytes + (size_t)i * 16), f);
#pragma unroll
      for (int q = 0; q < 8; ++q) acc[q] += wkk * f[q];
    }
  }
}

}  // namespace

// SHARED = false drops the shared-expert loads.  One unit's 9 expert-row loads are in flight at a time (plus the
// residual and shared rows of both units): two units' worth does not fit the 128 registers a 512-thread block leaves.
template <bool SHARED, bool FP8>
__global__ void __launch_bounds__(kRmsThreads, 1) ep_ll_combine_rmsnorm(const __grid_constant__ DevComm c,
                                                                        const __grid_constant__ EpLLCombineArgs a,
                                                                        const void* __restrict__ shared,
                                                                        const __grid_constant__ RmsNormArgs r) {
  __shared__ float s_warp[kRmsThreads / 32];
  const int tid = threadIdx.x, lane = tid & 31;
  const uint32_t upr = r.H / 8;
  const size_t row_bytes = (size_t)a.H * 2;
  BlockSync s = sync_begin(c, kDomEpLL, blockIdx.x);
  if (a.phase != EP_LL_RECV) sync_signal(c, s);
  sync_wait(c, s, blockIdx.x == 0 ? a.wait_stats : nullptr);

  // lane k holds the token's top-k entry k (every warp loads the same K entries, as in ep_ll_combine_kernel)
  auto load_route = [&](uint64_t t, long long& pos, float& w) {
    pos = -1;
    w = 0.f;
    if (lane < a.K && t < r.T) {
      pos = a.send_pos[t * a.K + lane];
      w = a.topk_weights[t * a.K + lane];
    }
  };
  long long pos;
  float w;
  load_route(blockIdx.x, pos, w);
  for (uint64_t t = blockIdx.x; t < r.T; t += gridDim.x) {
    long long next_pos;
    float next_w;
    load_route(t + gridDim.x, next_pos, next_w);
    const char* rowp[9];
    float wk[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      const long long pk = __shfl_sync(0xffffffffu, pos, k);
      wk[k] = __shfl_sync(0xffffffffu, w, k);
      rowp[k] = nullptr;
      if (k < a.K && pk >= 0) rowp[k] = c.heap[(int)(pk >> 32)] + a.x_off + (size_t)(pk & 0xffffffffll) * row_bytes;
    }
    uint4 res[kLLUnits], sh[kLLUnits];
    rmsnorm_load_residual<__nv_bfloat16>(res, t, r);
    if constexpr (SHARED) {
#pragma unroll
      for (int j = 0; j < kLLUnits; ++j) {
        const uint32_t u = j * kRmsThreads + tid;
        if (u < upr) sh[j] = ld_nc_v4(static_cast<const char*>(shared) + (t * upr + u) * 16);
      }
    }
    float v[kLLUnits][8];
#pragma unroll
    for (int j = 0; j < kLLUnits; ++j) {
      if (j * kRmsThreads >= (int)upr) break;  // block-uniform: the K > 9 tail shuffles
      const uint32_t u = j * kRmsThreads + tid;
      const bool valid = u < upr;
      uint4 x[9];
#pragma unroll
      for (int k = 0; k < 9; ++k)
        if (rowp[k] && valid) x[k] = ld_nc_v4(rowp[k] + (size_t)u * 16);
      float acc[8];
      ll_weighted_sum(acc, x, rowp, wk, valid, pos, w, a.K, c, a.x_off, row_bytes, u);
      if constexpr (SHARED) {
        float f[8];
        bf16x8_to_float(sh[j], f);
#pragma unroll
        for (int i = 0; i < 8; ++i) v[j][i] = round_to<__nv_bfloat16>(round_to<__nv_bfloat16>(acc[i]) + f[i]);
      } else {
#pragma unroll
        for (int i = 0; i < 8; ++i) v[j][i] = round_to<__nv_bfloat16>(acc[i]);
      }
    }
    rmsnorm_row_loaded<__nv_bfloat16, FP8>(v, res, t, r, s_warp);
    pos = next_pos;
    w = next_w;
  }
  sync_barrier_relaxed(c, s);  // nobody still reads my expert outputs when I return
  sync_end(s);
}

cudaError_t launch_ep_ll_combine_rmsnorm(const DevComm& c, const EpLLCombineArgs& a, const void* shared,
                                         const RmsNormArgs& r, bool fp8, int grid, cudaStream_t st) {
  if (a.phase == EP_LL_SEND || (uint32_t)a.H > (uint32_t)kLLUnits * kRmsThreads * 8) return cudaErrorInvalidValue;
  if (shared && fp8) UB_LAUNCH((ep_ll_combine_rmsnorm<true, true>), grid, kRmsThreads, 0, st, c, a, shared, r);
  else if (shared) UB_LAUNCH((ep_ll_combine_rmsnorm<true, false>), grid, kRmsThreads, 0, st, c, a, shared, r);
  else if (fp8) UB_LAUNCH((ep_ll_combine_rmsnorm<false, true>), grid, kRmsThreads, 0, st, c, a, shared, r);
  else UB_LAUNCH((ep_ll_combine_rmsnorm<false, false>), grid, kRmsThreads, 0, st, c, a, shared, r);
  return cudaGetLastError();
}

}  // namespace ub

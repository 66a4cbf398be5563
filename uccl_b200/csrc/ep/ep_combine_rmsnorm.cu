// EP combine fused with the residual add and RMSNorm that end an MoE layer, optionally quantised to e4m3 for the
// next layer's fp8 GEMM or dispatch:
//
//   combined     = bf16(0 + bias0 + bias1 + sum of the token's expert rows in ascending source rank)   (fp32)
//   residual_out = bf16(combined + residual)
//   out          = bf16(residual_out * rsqrt(mean(residual_out^2) + eps) * weight)   [-> e4m3 + scales]
//
// combined is exactly what ep_combine_kernel / the TMA combine write, but it is never stored: the row stays in
// registers and goes straight into the row epilogue of rmsnorm_row.cuh, the same one add_rmsnorm_kernel runs.  So
// the result is bitwise that of combine followed by add_rmsnorm_kernel, without the write and re-read of combined.
//
// Row-owned: block b owns token rows b, b + grid, ... and its kRmsThreads threads hold one row, unit
// k * kRmsThreads + threadIdx.x each.  One row is in flight per block, so a row's loads (its send_slot entries were
// fetched during the previous row) are all issued before the first add: residual, bias and every source rank's
// expert row, as many units at a time as registers allow.
#include "../kernels/launch.h"
#include "../kernels/rmsnorm_row.cuh"
#include "ep_buffer.h"
#include "ep_common.cuh"

namespace ub {

// NR = rank-count bucket (1, 2, 4, 8): the source loop unrolls to NR.  BIAS = false drops the bias loads.
// KB = units whose rows are in flight together: at most 12 16-byte loads (sources + biases) per thread, so that the
// kernel fits in the 128 registers a 512-thread block leaves without spilling.
template <int NR, bool BIAS, bool FP8>
__global__ void __launch_bounds__(kRmsThreads, 1) ep_combine_rmsnorm(const __grid_constant__ DevComm c,
                                                                     const __grid_constant__ EpCombineArgs a,
                                                                     const __grid_constant__ RmsNormArgs r) {
  constexpr int kLoads = NR + (BIAS ? 2 : 0);  // 16-byte loads per unit
  constexpr int KB = kLoads * kRmsUnits <= 12 ? kRmsUnits : (kLoads * 2 <= 12 ? 2 : 1);
  __shared__ float s_warp[kRmsThreads / 32];
  const int R = c.nranks, tid = threadIdx.x;
  const uint32_t upr = r.H / 8;
  const size_t row_bytes = (size_t)a.H * 2;
  BlockSync s = sync_begin(c, kDomEp, blockIdx.x);
  sync_barrier(c, s);  // every rank's expert outputs are in its combine arena

  auto load_slots = [&](uint64_t t, int (&sl)[NR]) {
#pragma unroll
    for (int q = 0; q < NR; ++q) sl[q] = (q < R && t < r.T) ? __ldg(a.send_slot + t * R + q) : -1;
  };
  int slot[NR];
  load_slots(blockIdx.x, slot);
  for (uint64_t t = blockIdx.x; t < r.T; t += gridDim.x) {
    int next[NR];
    load_slots(t + gridDim.x, next);
    const char* src[NR];
#pragma unroll
    for (int q = 0; q < NR; ++q) src[q] = c.heap[q] + a.x_off + (size_t)slot[q] * row_bytes;
    const char* b0 = BIAS && a.bias0 ? static_cast<const char*>(a.bias0) + t * row_bytes : nullptr;
    const char* b1 = BIAS && a.bias1 ? static_cast<const char*>(a.bias1) + t * row_bytes : nullptr;

    uint4 res[kRmsUnits];
    rmsnorm_load_residual<__nv_bfloat16>(res, t, r);
    float v[kRmsUnits][8];
#pragma unroll
    for (int k0 = 0; k0 < kRmsUnits; k0 += KB) {
      if (k0 * kRmsThreads >= (int)upr) break;  // block-uniform
      uint4 x[KB][NR], xb0[KB], xb1[KB];
#pragma unroll
      for (int j = 0; j < KB; ++j) {
        const uint32_t u = (k0 + j) * kRmsThreads + tid;
        if (u >= upr) continue;
        if constexpr (BIAS) {
          if (b0) xb0[j] = ld_nc_v4(b0 + (size_t)u * 16);
          if (b1) xb1[j] = ld_nc_v4(b1 + (size_t)u * 16);
        }
#pragma unroll
        for (int q = 0; q < NR; ++q)
          if (slot[q] >= 0) x[j][q] = ld_nc_v4(src[q] + (size_t)u * 16);
      }
#pragma unroll
      for (int j = 0; j < KB; ++j) {
        const uint32_t u = (k0 + j) * kRmsThreads + tid;
        if (u >= upr) continue;
        // the summation of ep_combine_kernel: fp32 from 0, bias0, bias1, then the sources in ascending rank
        float acc[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = 0.f;
        if constexpr (BIAS) {
          if (b0) {
            float f[8];
            bf16x8_to_float(xb0[j], f);
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[i] += f[i];
          }
          if (b1) {
            float f[8];
            bf16x8_to_float(xb1[j], f);
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[i] += f[i];
          }
        }
#pragma unroll
        for (int q = 0; q < NR; ++q) {
          if (slot[q] >= 0) {
            float f[8];
            bf16x8_to_float(x[j][q], f);
#pragma unroll
            for (int i = 0; i < 8; ++i) acc[i] += f[i];
          }
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) v[k0 + j][i] = round_to<__nv_bfloat16>(acc[i]);
      }
    }
    rmsnorm_row_loaded<__nv_bfloat16, FP8>(v, res, t, r, s_warp);
#pragma unroll
    for (int q = 0; q < NR; ++q) slot[q] = next[q];
  }
  sync_barrier_relaxed(c, s);  // nobody still reads my arena when I return
  sync_end(s);
}

template <int NR>
static cudaError_t launch_ep_combine_rmsnorm_nr(const DevComm& c, const EpCombineArgs& a, const RmsNormArgs& r,
                                                bool fp8, int grid, cudaStream_t st) {
  const bool bias = a.bias0 || a.bias1;
  if (bias && fp8) UB_LAUNCH((ep_combine_rmsnorm<NR, true, true>), grid, kRmsThreads, 0, st, c, a, r);
  else if (bias) UB_LAUNCH((ep_combine_rmsnorm<NR, true, false>), grid, kRmsThreads, 0, st, c, a, r);
  else if (fp8) UB_LAUNCH((ep_combine_rmsnorm<NR, false, true>), grid, kRmsThreads, 0, st, c, a, r);
  else UB_LAUNCH((ep_combine_rmsnorm<NR, false, false>), grid, kRmsThreads, 0, st, c, a, r);
  return cudaGetLastError();
}

cudaError_t launch_ep_combine_rmsnorm(const DevComm& c, const EpCombineArgs& a, const RmsNormArgs& r, bool fp8,
                                      int grid, cudaStream_t st) {
  switch (c.nranks) {
    case 1: return launch_ep_combine_rmsnorm_nr<1>(c, a, r, fp8, grid, st);
    case 2: return launch_ep_combine_rmsnorm_nr<2>(c, a, r, fp8, grid, st);
    case 3: case 4: return launch_ep_combine_rmsnorm_nr<4>(c, a, r, fp8, grid, st);
    default: return launch_ep_combine_rmsnorm_nr<8>(c, a, r, fp8, grid, st);
  }
}

}  // namespace ub

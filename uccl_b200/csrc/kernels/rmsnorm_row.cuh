// Row epilogue of the fused layer tails: residual add, RMSNorm and the optional per-128-channel e4m3 cast of one
// row held in registers by a block of kRmsThreads threads.  Shared by allreduce_rmsnorm.cu (TP / SP tails and the
// local add_rmsnorm_kernel) and ep/ep_combine_rmsnorm.cu (EP combine tail).  Every caller uses the identical
// thread -> element mapping (unit k * kRmsThreads + threadIdx.x of the row), so their results are bitwise equal.
// U (default kRmsUnits) is the number of units a thread holds: a caller whose rows are shorter (the low-latency EP
// combine, H <= 8192, needs 2) passes fewer and saves the registers of the units it can never have.
#pragma once
#include "fp8_quant.cuh"
#include "reduce.cuh"
#include "types.h"

namespace ub {

template <typename T>
__device__ __forceinline__ float round_to(float v) {
  return to_acc<float, T>(from_acc<T, float>(v));
}

// Load half: the thread's units of the residual row.  Callers that also load the values to normalise issue both
// before the first use, so a row costs one memory round trip instead of two.
template <typename T, int U = kRmsUnits>
__device__ __forceinline__ void rmsnorm_load_residual(uint4 (&res)[U], uint64_t row, const RmsNormArgs& r) {
  const uint32_t upr = r.H / 8;  // 16-byte units per row
  const uint64_t base = row * upr;
#pragma unroll
  for (int k = 0; k < U; ++k) {
    const uint32_t u = k * kRmsThreads + threadIdx.x;
    if (u < upr) res[k] = ld_v4(static_cast<const char*>(r.residual) + (base + u) * 16);
  }
}

// Compute half.  v[k] holds the reduced values (already rounded to T) of unit k * kRmsThreads + threadIdx.x of the
// row, res[k] the same units of the residual (rmsnorm_load_residual).  The whole residual row is loaded before
// anything is stored, and every thread only stores the units it loaded, so residual_out may alias residual.  All
// kRmsThreads threads of the block must call it.
template <typename T, bool FP8, int U = kRmsUnits>
__device__ __forceinline__ void rmsnorm_row_loaded(float (&v)[U][8], const uint4 (&res)[U], uint64_t row,
                                                   const RmsNormArgs& r, float* s_warp) {
  const int tid = threadIdx.x;
  const uint32_t upr = r.H / 8;
  const uint64_t base = row * upr;
  // residual add, rounded to T; sum of squares of the rounded values in a fixed order
  float ss = 0.f;
#pragma unroll
  for (int k = 0; k < U; ++k) {
    const uint32_t u = k * kRmsThreads + tid;
    if (u < upr) {
      Vec16<T, kSum> rv;
      rv.init(res[k]);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        rv.a[i] = round_to<T>(v[k][i] + rv.a[i]);
        v[k][i] = rv.a[i];
        ss = __fmaf_rn(rv.a[i], rv.a[i], ss);
      }
      st_v4(static_cast<char*>(r.residual_out) + (base + u) * 16, rv.pack_same());
    }
  }
  // block sum: butterfly inside each warp, then the warp partials in warp order
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  if ((tid & 31) == 0) s_warp[tid >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int w = 0; w < kRmsThreads / 32; ++w) tot += s_warp[w];
  __syncthreads();  // s_warp is reused by the next row
  const float inv = rsqrtf(__fdiv_rn(tot, (float)r.H) + r.eps);

#pragma unroll
  for (int k = 0; k < U; ++k) {
    if (k * kRmsThreads >= (int)upr) break;  // block-uniform: the fp8 path shuffles below
    const uint32_t u = k * kRmsThreads + tid;
    const bool valid = u < upr;
    Vec16<T, kSum> y;
#pragma unroll
    for (int i = 0; i < 8; ++i) y.a[i] = 0.f;
    if (valid) {
      Vec16<T, kSum> w;
      w.init(ld_nc_v4(static_cast<const char*>(r.weight) + (uint64_t)u * 16));
#pragma unroll
      for (int i = 0; i < 8; ++i) y.a[i] = round_to<T>(__fmul_rn(__fmul_rn(v[k][i], inv), w.a[i]));
    }
    if constexpr (!FP8) {
      if (valid) st_v4(static_cast<char*>(r.out) + (base + u) * 16, y.pack_same());
    } else {
      // one 128-channel group = 16 consecutive units = 16 consecutive lanes (kRmsThreads and upr are multiples of 16)
      float amax = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) amax = fmaxf(amax, fabsf(y.a[i]));
#pragma unroll
      for (int o = 1; o < 16; o <<= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
      float scale, scale_inv;
      fp8_group_scale_torch(amax, scale, scale_inv);
      uint2 q;
      q.x = pack4_e4m3(y.a[0] * scale, y.a[1] * scale, y.a[2] * scale, y.a[3] * scale);
      q.y = pack4_e4m3(y.a[4] * scale, y.a[5] * scale, y.a[6] * scale, y.a[7] * scale);
      if (valid) {
        st_v2(static_cast<char*>(r.out) + (base + u) * 8, q);
        if ((tid & 15) == 0) r.out_scales[row * (r.H / 128) + u / 16] = scale_inv;
      }
    }
  }
}

// Both halves back to back, for callers whose values are already in registers.
template <typename T, bool FP8>
__device__ __forceinline__ void rmsnorm_row(float (&v)[kRmsUnits][8], uint64_t row, const RmsNormArgs& r,
                                            float* s_warp) {
  uint4 res[kRmsUnits];
  rmsnorm_load_residual<T>(res, row, r);
  rmsnorm_row_loaded<T, FP8>(v, res, row, r, s_warp);
}

}  // namespace ub

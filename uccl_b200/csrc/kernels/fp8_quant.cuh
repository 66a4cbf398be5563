// Per-128-channel e4m3 quantiser shared by the expert-parallel dispatch kernels (ep/) and the fused
// all-reduce + RMSNorm epilogue (allreduce_rmsnorm.cu).  Bit-identical to ep.utils.per_token_cast_to_fp8.
#pragma once
#include "prims.cuh"

namespace ub {

__device__ __forceinline__ uint32_t pack4_e4m3(float a, float b, float c, float d) {
  __nv_fp8x2_storage_t lo = __nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, __NV_E4M3);
  __nv_fp8x2_storage_t hi = __nv_cvt_float2_to_fp8x2(make_float2(c, d), __NV_SATFINITE, __NV_E4M3);
  return (uint32_t)lo | ((uint32_t)hi << 16);
}


// scale / inverse scale of one 128-channel group from its amax (bit-identical to the torch reference
// `amax.clamp(1e-4) / 448`; round_scale: power-of-two inverse scale, UE8M0 compatible)
__device__ __forceinline__ void fp8_group_scale(float amax, int round_scale, float& scale, float& scale_inv) {
  amax = fmaxf(amax, 1e-4f);
  if (round_scale) {
    const float raw = amax * (1.0f / 448.0f);
    int ex = ((__float_as_int(raw) >> 23) & 0xff) - 127;
    if ((__float_as_int(raw) & 0x7fffff) != 0) ex += 1;
    scale_inv = __int_as_float((ex + 127) << 23);
    scale = __int_as_float((127 - ex) << 23);
  } else {
    scale = 448.0f / amax;
    scale_inv = __fdiv_rn(amax, 448.0f);
  }
}

// fp8_group_scale(amax, 0, ...) with the scale rounded exactly as per_token_cast_to_fp8 computes it: torch
// evaluates `448.0 / amax` as reciprocal(amax) * 448, two roundings that differ from one correctly rounded
// division in the last bit for about a quarter of all amax values (and then, rarely, in an e4m3 byte).
__device__ __forceinline__ void fp8_group_scale_torch(float amax, float& scale, float& scale_inv) {
  amax = fmaxf(amax, 1e-4f);
  scale = __fmul_rn(__frcp_rn(amax), 448.0f);
  scale_inv = __fdiv_rn(amax, 448.0f);
}

}  // namespace ub

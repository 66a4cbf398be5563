// All-reduce (sum) fused with the residual add and RMSNorm that follow every row-parallel GEMM of a
// tensor-parallel transformer, optionally quantised to e4m3 for an fp8 GEMM or an EP dispatch:
//
//   x            = sum_r x_r                          (fp32 in rank order, rounded once; in place)
//   residual_out = T(x + residual)
//   out          = T(residual_out * rsqrt(mean(residual_out^2) + eps) * weight)   [-> e4m3 + scales]
//
//   ar_oneshot_rmsnorm<T, MC, FP8>  the one-shot LL all-reduce (allreduce_impl.cuh) with row-owned phases: block b
//                                   publishes and reduces rows b, b + grid, ... and runs the row epilogue on the
//                                   reduced row while it is still in registers.  No barrier, no extra HBM pass.
//   add_rmsnorm_kernel<T, FP8>      the same row epilogue on an already reduced x (the unfused path behind the
//                                   two-shot / staged / NVLS all-reduce or the barrier-based reduce-scatter, and
//                                   one-rank communicators).
//   rs_ll_rmsnorm<T, FP8>           sequence-parallel variant: the LL reduce-scatter of ll_exchange.cuh with a
//                                   row-owned phase 2; x is [T, H] summed over ranks, and rank r keeps, reduces and
//                                   normalises only its T / n rows (residual, residual_out and out are that shard).
// All run the identical epilogue (rmsnorm_row.cuh) with the identical thread -> element mapping, so their results
// are bitwise equal.
#include "allreduce_impl.cuh"
#include "ll_exchange.cuh"
#include "rmsnorm_row.cuh"

namespace ub {

// Fused path: the one-shot LL all-reduce of allreduce_impl.cuh (same epoch words, packet slots and spin sites)
// with row-owned phases.  A block publishes exactly the rows it later reduces, with the same thread -> unit
// mapping, so storing the sum over x in place never races with another block still publishing x.
// The grid must not exceed the one-shot's: with virtual ranks every rank's blocks have to be resident at once.
template <typename T, bool MC, bool FP8>
__global__ void __launch_bounds__(kRmsThreads) ar_oneshot_rmsnorm(const __grid_constant__ DevComm c,
                                                                  const __grid_constant__ CollArgs a,
                                                                  const __grid_constant__ RmsNormArgs r) {
  __shared__ float s_warp[kRmsThreads / 32];
  uint32_t* misc = reinterpret_cast<uint32_t*>(c.heap[c.rank] + a.misc_off);
  const uint32_t flag = ll_begin(misc);
  const uint64_t parity_off = ll_parity_off(a, flag);
  const uint32_t upr = r.H / 8;
  const int n = c.nranks, rank = c.rank, tid = threadIdx.x;

  for (uint64_t row = blockIdx.x; row < r.T; row += gridDim.x)
    ll_publish<MC>(c, a, flag, parity_off, row * upr + tid, (row + 1) * upr, kRmsThreads);

  const char* my_ll = c.heap[rank] + parity_off;
  char* x = static_cast<char*>(r.x);
  for (uint64_t row = blockIdx.x; row < r.T; row += gridDim.x) {
    float v[kRmsUnits][8];
#pragma unroll
    for (int k = 0; k < kRmsUnits; ++k) {
      const uint32_t ur = k * kRmsThreads + tid;
      if (ur >= upr) continue;
      const uint64_t u = row * upr + ur;
      Vec16<T, kSum> acc;
      for (int s = 0; s < n; ++s) {
        const uint4 d = s == rank ? ld_v4(x + u * 16) : ll_recv(c, my_ll, s, u, flag);
        if (s == 0) acc.init(d);
        else acc.accum(d);
      }
      const uint4 sum = acc.pack_same();
      st_v4(x + u * 16, sum);
      Vec16<T, kSum> rounded;
      rounded.init(sum);
#pragma unroll
      for (int i = 0; i < 8; ++i) v[k][i] = rounded.a[i];
    }
    rmsnorm_row<T, FP8>(v, row, r, s_warp);
  }
  ll_end(misc, flag);
}

template <typename T, bool FP8>
__global__ void __launch_bounds__(kRmsThreads) add_rmsnorm_kernel(const __grid_constant__ RmsNormArgs r) {
  __shared__ float s_warp[kRmsThreads / 32];
  const uint32_t upr = r.H / 8;
  const char* x = static_cast<const char*>(r.x);
  for (uint64_t row = blockIdx.x; row < r.T; row += gridDim.x) {
    float v[kRmsUnits][8];
#pragma unroll
    for (int k = 0; k < kRmsUnits; ++k) {
      const uint32_t ur = k * kRmsThreads + threadIdx.x;
      if (ur >= upr) continue;
      Vec16<T, kSum> xv;
      xv.init(ld_v4(x + (row * upr + ur) * 16));
#pragma unroll
      for (int i = 0; i < 8; ++i) v[k][i] = xv.a[i];
    }
    rmsnorm_row<T, FP8>(v, row, r, s_warp);
  }
}

// Fused sequence-parallel path: rs_ll_kernel's phases and protocol (ll_begin / ll_end of ll_exchange.cuh: the same
// epoch words and parity slots as every other LL collective and the one-shot all-reduce).  a.in = the whole x,
// a.bytes = one rank's piece (r.T * H * sizeof(T), with r.T = T / n rows); r.x = my own piece of x.
// Phase 1 pushes the peers' pieces and never reads my own, so phase 2 may store the sum over it: every unit of my
// piece is loaded and stored by one thread only.  Blocks past the last row only push: the grid is rs_ll_kernel's,
// which keeps phase 1 wide when a rank has one or two rows, and never exceeds it (co-residency of virtual ranks).
template <typename T, bool FP8>
__global__ void __launch_bounds__(kRmsThreads) rs_ll_rmsnorm(const __grid_constant__ DevComm c,
                                                             const __grid_constant__ CollArgs a,
                                                             const __grid_constant__ RmsNormArgs r) {
  __shared__ float s_warp[kRmsThreads / 32];
  const LLCtx l = ll_begin(c, a);
  const uint32_t upr = r.H / 8;
  const int n = c.nranks, rank = c.rank, tid = threadIdx.x;

  ll_scatter_pieces(c, a, l, (uint64_t)r.T * upr);

  const char* my_ll = c.heap[rank] + l.parity_off;
  char* x = static_cast<char*>(r.x);
  for (uint64_t row = blockIdx.x; row < r.T; row += gridDim.x) {
    float v[kRmsUnits][8];
#pragma unroll
    for (int k = 0; k < kRmsUnits; ++k) {
      const uint32_t ur = k * kRmsThreads + tid;
      if (ur >= upr) continue;
      const uint64_t u = row * upr + ur;  // unit of my piece = unit of every peer's packet slot
      Vec16<T, kSum> acc;
      for (int s = 0; s < n; ++s) {
        const uint4 d =
            s == rank ? ld_v4(x + u * 16) : ll_get(c, my_ll + (uint64_t)s * kLLSlotBytes + u * 32, l.flag, s);
        if (s == 0) acc.init(d);
        else acc.accum(d);
      }
      const uint4 sum = acc.pack_same();
      st_v4(x + u * 16, sum);
      Vec16<T, kSum> rounded;
      rounded.init(sum);
#pragma unroll
      for (int i = 0; i < 8; ++i) v[k][i] = rounded.a[i];
    }
    rmsnorm_row<T, FP8>(v, row, r, s_warp);
  }
  ll_end(l);
}

template <typename T, bool FP8>
static cudaError_t launch_rms_typed(int algo, const DevComm& c, const CollArgs& a, const RmsNormArgs& r, int grid,
                                    cudaStream_t st) {
  switch (algo) {
    case 0: UB_LAUNCH((add_rmsnorm_kernel<T, FP8>), grid, kRmsThreads, 0, st, r); break;
    case AR_ONESHOT_LL: UB_LAUNCH((ar_oneshot_rmsnorm<T, false, FP8>), grid, kRmsThreads, 0, st, c, a, r); break;
    case AR_ONESHOT_MC: UB_LAUNCH((ar_oneshot_rmsnorm<T, true, FP8>), grid, kRmsThreads, 0, st, c, a, r); break;
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

cudaError_t launch_allreduce_rmsnorm(int algo, int dtype, bool fp8, const DevComm& c, const CollArgs& a,
                                     const RmsNormArgs& r, int grid, cudaStream_t st) {
  switch (dtype) {
    case kBF16:
      return fp8 ? launch_rms_typed<__nv_bfloat16, true>(algo, c, a, r, grid, st)
                 : launch_rms_typed<__nv_bfloat16, false>(algo, c, a, r, grid, st);
    case kF16:
      return fp8 ? launch_rms_typed<__half, true>(algo, c, a, r, grid, st)
                 : launch_rms_typed<__half, false>(algo, c, a, r, grid, st);
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t launch_reduce_scatter_rmsnorm(int dtype, bool fp8, const DevComm& c, const CollArgs& a,
                                          const RmsNormArgs& r, int grid, cudaStream_t st) {
  switch (dtype) {
    case kBF16:
      if (fp8) UB_LAUNCH((rs_ll_rmsnorm<__nv_bfloat16, true>), grid, kRmsThreads, 0, st, c, a, r);
      else UB_LAUNCH((rs_ll_rmsnorm<__nv_bfloat16, false>), grid, kRmsThreads, 0, st, c, a, r);
      break;
    case kF16:
      if (fp8) UB_LAUNCH((rs_ll_rmsnorm<__half, true>), grid, kRmsThreads, 0, st, c, a, r);
      else UB_LAUNCH((rs_ll_rmsnorm<__half, false>), grid, kRmsThreads, 0, st, c, a, r);
      break;
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

}  // namespace ub

// Device code shared by the register-path (ep_kernels.cu) and the TMA-pipelined (ep_tma_kernels.cu)
// expert-parallel kernels: bf16 -> fp32 helper, the per-128-channel quantiser (kernels/fp8_quant.cuh)
// and the count-exchange prologue of a non-cached dispatch.
#pragma once
#include "../kernels/fp8_quant.cuh"
#include "../kernels/prims.cuh"
#include "ep_types.h"

namespace ub {

__device__ __forceinline__ void bf16x8_to_float(const uint4& v, float (&f)[8]) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 p = __bfloat1622float2(h[i]);
    f[2 * i] = p.x;
    f[2 * i + 1] = p.y;
  }
}

// Count exchange of a non-cached dispatch (all threads of the block call it; the block has at
// least kMaxRanks * kMaxRanks threads).  On return s_base[r] = first slot of my tokens inside rank
// r's arena, *s_abort != 0 if some arena would overflow (same decision on every rank) and
// *s_recv_total = tokens this rank receives.  Block 0 also publishes the receive counts.
// Cached dispatches only rendezvous (the peers' arenas may be overwritten from here on).
__device__ __forceinline__ void ep_dispatch_prologue(const DevComm& c, const EpDispatchArgs& a, BlockSync& s,
                                                     int (*s_M)[kMaxRanks], int* s_base, int* s_abort,
                                                     int* s_recv_total) {
  const int R = c.nranks, me = c.rank;
  const int tid = threadIdx.x;
  const int E_local = a.E / R;
  if (!a.cached) {
    // ---- phase 0: all-gather the R x R count matrix (each block keeps a private copy so that
    //      only same-index blocks of different ranks need to synchronise)
    if (tid < R * R) {
      const int dst = tid / R, j = tid % R;
      int* p = reinterpret_cast<int*>(c.heap[dst] + a.cnt_tab_off) + ((size_t)blockIdx.x * kMaxRanks + me) * kMaxRanks + j;
      *p = a.tokens_per_rank[j];
    }
    if (blockIdx.x == 0) {
      for (int i = tid; i < R * E_local; i += blockDim.x) {
        const int dst = i / E_local, e = i % E_local;
        int* p = reinterpret_cast<int*>(c.heap[dst] + a.exp_tab_off) + (size_t)me * kEpMaxLocalExperts + e;
        *p = a.tokens_per_expert[dst * E_local + e];
      }
    }
    sync_barrier(c, s);
    const int* my_tab = reinterpret_cast<const int*>(c.heap[me] + a.cnt_tab_off) + (size_t)blockIdx.x * kMaxRanks * kMaxRanks;
    if (tid < R * R) s_M[tid / R][tid % R] = my_tab[(tid / R) * kMaxRanks + (tid % R)];
    __syncthreads();
    if (tid < R) {
      int base = 0, tot = 0;
      for (int q = 0; q < R; ++q) {
        if (q < me) base += s_M[q][tid];
        tot += s_M[q][tid];
      }
      s_base[tid] = base;
      if (tot > a.arena.capacity) *s_abort = 1;  // identical decision on every rank (same matrix)
      if (tid == me) *s_recv_total = tot;
    }
    __syncthreads();
    if (blockIdx.x == 0) {
      if (a.rank_prefix && tid < R * R) a.rank_prefix[tid] = s_M[tid / R][tid % R];
      const int* exp_tab = reinterpret_cast<const int*>(c.heap[me] + a.exp_tab_off);
      for (int e = tid; e < E_local; e += blockDim.x) {
        int tot = 0;
        for (int q = 0; q < R; ++q) tot += exp_tab[(size_t)q * kEpMaxLocalExperts + e];
        const int al = a.expert_alignment > 1 ? a.expert_alignment : 1;
        tot = (tot + al - 1) / al * al;
        a.dev_counts[1 + e] = tot;
        if (a.host_counts) a.host_counts[1 + e] = tot;
      }
      __syncthreads();
      if (tid == 0) {
        const int v = *s_abort ? -2 : *s_recv_total;
        a.dev_counts[0] = v;
        if (a.host_counts) {
          __threadfence_system();
          a.host_counts[0] = v;
          __threadfence_system();
        }
      }
    }
  } else {
    sync_barrier_relaxed(c, s);  // peers have entered this dispatch: their arena may be overwritten
    if (tid < R) s_base[tid] = 0;
    __syncthreads();
  }

}

}  // namespace ub

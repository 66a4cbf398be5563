// Device primitives for sm_90a communication kernels.
//
// What the reference provides here (behaviour, not code):
//   * ep/include/ep_utils.cuh:259-395  L1-no-allocate loads/stores, sys-scope acquire/release
//   * ep/include/ep_utils.cuh:447-585  TMA 1-D bulk copies + mbarrier helpers
//   * experimental/lite/core/switch_channel_device.hpp:42-290  multimem.ld_reduce/st/red
//   * experimental/lite/core/semaphore_device.hpp:66-145  device semaphores with spin caps
// This file is the Hopper-native equivalent: every peer access is a plain global
// (or multimem) instruction on an NVLink-mapped VA from the symmetric heap.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "types.h"

namespace ub {

// ---------------------------------------------------------------- memory ops
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint64_t ld_acquire_sys(const uint64_t* p) {
  uint64_t v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_relaxed_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_volatile(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void st_release_sys(uint64_t* p, uint64_t v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void st_relaxed_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void red_add_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("red.release.sys.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void red_add_relaxed_sys(uint32_t* p, uint32_t v) {
  asm volatile("red.relaxed.sys.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_gpu(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_gpu(uint32_t* p, uint32_t v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void fence_acq_rel_sys() { asm volatile("fence.acq_rel.sys;" ::: "memory"); }
__device__ __forceinline__ void fence_acq_rel_gpu() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }

// 16-byte streaming accesses (no L1 allocation; peer data is never re-read).
__device__ __forceinline__ uint4 ld_nc_v4(const void* p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}
// coherent 16-byte load (data another GPU may have just written; ordered by an acquire)
__device__ __forceinline__ uint4 ld_v4(const void* p) {
  uint4 v;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
__device__ __forceinline__ uint4 ld_volatile_v4(const void* p) {
  uint4 v;
  asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
__device__ __forceinline__ void st_v4(void* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y),
               "r"(v.z), "r"(v.w)
               : "memory");
}
__device__ __forceinline__ void st_v2(void* p, const uint2& v) {
  asm volatile("st.global.L1::no_allocate.v2.u32 [%0], {%1,%2};" ::"l"(p), "r"(v.x), "r"(v.y) : "memory");
}
__device__ __forceinline__ uint2 ld_nc_v2(const void* p) {
  uint2 v;
  asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p));
  return v;
}

// ------------------------------------------------------------- NVLS multimem
// multimem ops are issued on the multicast VA; the NVSwitch performs the
// reduction (ld_reduce) or the replication (st) in the fabric.
template <typename T>
struct Multimem;  // ld_reduce_add(const void* mc) -> uint4 ; specialised per dtype

__device__ __forceinline__ void multimem_st_v4(void* mc, const uint4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "r"(v.x), "r"(v.y),
               "r"(v.z), "r"(v.w)
               : "memory");
}
__device__ __forceinline__ void multimem_st_v2(void* mc, const uint2& v) {
  asm volatile("multimem.st.relaxed.sys.global.v2.f32 [%0], {%1,%2};" ::"l"(mc), "r"(v.x), "r"(v.y)
               : "memory");
}
__device__ __forceinline__ void multimem_red_add_u32(void* mc, uint32_t v) {
  asm volatile("multimem.red.relaxed.sys.global.add.u32 [%0], %1;" ::"l"(mc), "r"(v) : "memory");
}
__device__ __forceinline__ void multimem_red_add_release_u32(void* mc, uint32_t v) {
  asm volatile("multimem.red.release.sys.global.add.u32 [%0], %1;" ::"l"(mc), "r"(v) : "memory");
}

#define UB_MM_LDRED(NAME, PTXOP)                                                      \
  __device__ __forceinline__ uint4 NAME(const void* mc) {                             \
    uint4 v;                                                                          \
    asm volatile("multimem.ld_reduce.relaxed.sys.global." PTXOP " {%0,%1,%2,%3}, [%4];" \
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)                         \
                 : "l"(mc)                                                            \
                 : "memory");                                                         \
    return v;                                                                         \
  }
UB_MM_LDRED(mm_ldred_add_f32, "add.v4.f32")
UB_MM_LDRED(mm_ldred_add_bf16, "add.acc::f32.v4.bf16x2")
UB_MM_LDRED(mm_ldred_add_f16, "add.acc::f32.v4.f16x2")
UB_MM_LDRED(mm_ldred_min_bf16, "min.v4.bf16x2")
UB_MM_LDRED(mm_ldred_max_bf16, "max.v4.bf16x2")
UB_MM_LDRED(mm_ldred_min_f16, "min.v4.f16x2")
UB_MM_LDRED(mm_ldred_max_f16, "max.v4.f16x2")
#undef UB_MM_LDRED

// ------------------------------------------------------- TMA 1-D bulk + mbarrier
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t phase) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(phase)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t phase) {
  while (!mbar_try_wait(bar, phase)) {
  }
}
// global -> shared bulk copy (bytes % 16 == 0, 16-byte aligned both sides); completes on `bar`.
__device__ __forceinline__ void tma_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(smem_dst)),
      "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
// shared -> global bulk copy (dst may be a peer-mapped VA); tracked by bulk async-groups.
__device__ __forceinline__ void tma_store_1d(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst),
               "r"(smem_u32(smem_src)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
// make generic-proxy smem writes visible to the async proxy (before a bulk store)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// ------------------------------------------------------------ spin with timeout
// Every spin in this library goes through SpinGuard so that a lost peer turns
// into a diagnosable trap instead of a hung GPU (reference: device timeouts that
// printf+trap, ep/src/intranode.cu:333-339).
struct SpinGuard {
  uint64_t t0;
  uint64_t limit;
  uint32_t n;
  __device__ __forceinline__ explicit SpinGuard(uint64_t timeout_ns) : t0(0), limit(timeout_ns), n(0) {}
  __device__ __forceinline__ bool expired() {
    if (((++n) & 0x3ff) != 0 || limit == 0) return false;
    uint64_t now = globaltimer_ns();
    if (t0 == 0) {
      t0 = now;
      return false;
    }
    return (now - t0) > limit;
  }
};

static __device__ __noinline__ void comm_abort(const DevComm& c, int code, int a, int b) {
  printf("[uccl_b200] rank %d block %d thread %d: spin timeout (site %d, peer/info %d, want %d)\n", c.rank,
         (int)blockIdx.x, (int)threadIdx.x, code, a, b);
  if (c.err) *c.err = 0x80000000u | (uint32_t)code;
  __threadfence_system();
  __trap();
}

// --------------------------------------------------------------- in-kernel tracing
// NPKit-style device timeline (reference: experimental/lite/core/npkit.hpp:30-60 stamps
// clock64() events at compile time).  Here it is a runtime switch: when the communicator has a
// trace buffer, thread 0 of every block appends {globaltimer, code|block|aux} -- every cross-rank
// barrier is stamped, so wait time vs copy time per block falls out of any kernel for free.
__device__ __forceinline__ void trace_event(const DevComm& c, uint32_t code, uint32_t aux) {
  if (c.trace == nullptr || threadIdx.x != 0) return;
  const unsigned long long idx = atomicAdd(c.trace, 1ull);
  if (idx < c.trace_cap) {
    c.trace[2 + 2 * idx] = globaltimer_ns();
    c.trace[3 + 2 * idx] = ((unsigned long long)code << 48) | ((unsigned long long)(blockIdx.x & 0xffff) << 32) | aux;
  }
}

// ------------------------------------------------------- cross-rank block barrier
// Slot layout inside every heap: sig[domain][block][src_rank] (u32, single writer each).
// Epochs are monotonic so no reset is ever needed; the local epoch of (domain, block)
// lives at epoch[domain][block] and is read once at kernel start (graph-replay safe).
struct BlockSync {
  uint32_t e;      // epoch value used by the *next* barrier
  uint32_t* my_sig;   // &my_heap.sig[domain][block][0]
  uint32_t* epoch_ptr;
  uint64_t sig_block_off;  // byte offset of sig[domain][block][0] inside a heap
};

__device__ __forceinline__ BlockSync sync_begin(const DevComm& c, int domain, int block) {
  BlockSync s;
  uint64_t idx = ((uint64_t)domain * kMaxSyncBlocks + block);
  s.sig_block_off = c.sig_off + idx * kMaxRanks * sizeof(uint32_t);
  s.my_sig = reinterpret_cast<uint32_t*>(c.heap[c.rank] + s.sig_block_off);
  s.epoch_ptr = reinterpret_cast<uint32_t*>(c.heap[c.rank] + c.epoch_off) + idx;
  s.e = ld_volatile(s.epoch_ptr) + 1;
  trace_event(c, TR_KERNEL_BEGIN, (uint32_t)domain);
  return s;
}

// All threads of the block must call. Orders all prior writes of the block (to any
// rank) before the barrier and all later reads after it.
__device__ __forceinline__ void sync_barrier(const DevComm& c, BlockSync& s) {
  __syncthreads();
  trace_event(c, TR_BARRIER_ENTER, s.e);
  const int t = threadIdx.x;
  if (t < c.nranks && t != c.rank) {
    uint32_t* peer_slot = reinterpret_cast<uint32_t*>(c.heap[t] + s.sig_block_off) + c.rank;
    st_release_sys(peer_slot, s.e);
    SpinGuard g(c.timeout_ns);
    while ((int32_t)(ld_acquire_sys(s.my_sig + t) - s.e) < 0) {
      if (g.expired()) comm_abort(c, 1, t, (int)s.e);
    }
  }
  s.e += 1;
  __syncthreads();
  trace_event(c, TR_BARRIER_EXIT, s.e - 1);
}
// Split barrier for kernels that are cut into a SEND and a RECV launch (EP low-latency hooks):
// sync_signal publishes "my writes up to here are done" to every peer without waiting, sync_wait (same
// block index, possibly a later kernel) blocks until every peer has published the same epoch.
// sync_signal does NOT advance the epoch: the kernel that signals stores epoch e-1 in sync_end, the
// kernel that waits re-reads it, waits for e and stores e.
__device__ __forceinline__ void sync_signal(const DevComm& c, BlockSync& s) {
  __syncthreads();
  const int t = threadIdx.x;
  if (t < c.nranks && t != c.rank) {
    uint32_t* peer_slot = reinterpret_cast<uint32_t*>(c.heap[t] + s.sig_block_off) + c.rank;
    st_release_sys(peer_slot, s.e);
  }
}
// wait_cycles (optional, [nranks] int64): clock cycles thread t spent waiting for rank t are added to it
__device__ __forceinline__ void sync_wait(const DevComm& c, BlockSync& s, long long* wait_cycles = nullptr) {
  const int t = threadIdx.x;
  trace_event(c, TR_BARRIER_ENTER, s.e);
  if (t < c.nranks && t != c.rank) {
    const long long t0 = clock64();
    SpinGuard g(c.timeout_ns);
    while ((int32_t)(ld_acquire_sys(s.my_sig + t) - s.e) < 0) {
      if (g.expired()) comm_abort(c, 3, t, (int)s.e);
    }
    if (wait_cycles) atomicAdd(reinterpret_cast<unsigned long long*>(wait_cycles + t), (unsigned long long)(clock64() - t0));
  }
  s.e += 1;
  __syncthreads();
  trace_event(c, TR_BARRIER_EXIT, s.e - 1);
}

// Barrier that also all-gathers two 64-bit words per rank (e.g. the heap offsets of this
// rank's input / output buffers) between same-index blocks.  `sh` is shared memory for
// 2 * kMaxRanks words: sh[r] = word0 of rank r, sh[kMaxRanks + r] = word1 of rank r.
// Lets zero-copy kernels work even when ranks allocated their symmetric buffers at different
// offsets (e.g. Python GC freed blocks in a different order on different ranks).
__device__ __forceinline__ void sync_exchange(const DevComm& c, BlockSync& s, int domain, uint64_t w0, uint64_t w1,
                                              uint64_t* sh) {
  const int t = threadIdx.x;
  const uint64_t idx = ((uint64_t)domain * kMaxSyncBlocks + blockIdx.x) * kMaxRanks;
  if (t < c.nranks && t != c.rank) {
    uint64_t* p = reinterpret_cast<uint64_t*>(c.heap[t] + c.xchg_off + (idx + c.rank) * 16);
    p[0] = w0;
    p[1] = w1;  // ordered before the signal by the release store of the same thread below
  }
  sync_barrier(c, s);
  if (t < c.nranks) {
    if (t == c.rank) {
      sh[t] = w0;
      sh[kMaxRanks + t] = w1;
    } else {
      const volatile uint64_t* p = reinterpret_cast<const volatile uint64_t*>(c.heap[c.rank] + c.xchg_off + (idx + t) * 16);
      sh[t] = p[0];
      sh[kMaxRanks + t] = p[1];
    }
  }
  __syncthreads();
}
__device__ __forceinline__ bool all_equal(const uint64_t* sh, int n) {
  bool same = true;
  for (int r = 1; r < n; ++r) same = same && (sh[r] == sh[0]);
  return same;
}

// Relaxed variant: only a rendezvous, no data ordering (cheaper: no release fence).
__device__ __forceinline__ void sync_barrier_relaxed(const DevComm& c, BlockSync& s) {
  __syncthreads();
  trace_event(c, TR_BARRIER_ENTER, s.e);
  const int t = threadIdx.x;
  if (t < c.nranks && t != c.rank) {
    uint32_t* peer_slot = reinterpret_cast<uint32_t*>(c.heap[t] + s.sig_block_off) + c.rank;
    st_relaxed_sys(peer_slot, s.e);
    SpinGuard g(c.timeout_ns);
    while ((int32_t)(ld_relaxed_sys(s.my_sig + t) - s.e) < 0) {
      if (g.expired()) comm_abort(c, 2, t, (int)s.e);
    }
  }
  s.e += 1;
  __syncthreads();
  trace_event(c, TR_BARRIER_EXIT, s.e - 1);
}
__device__ __forceinline__ void sync_end(BlockSync& s) {
  if (threadIdx.x == 0) *reinterpret_cast<volatile uint32_t*>(s.epoch_ptr) = s.e - 1;
}

// ------------------------------------------------------------------ warp helpers
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "elect.sync _|p, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(pred));
  return pred != 0;
}

}  // namespace ub

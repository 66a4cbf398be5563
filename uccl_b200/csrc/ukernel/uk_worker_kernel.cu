// Persistent worker kernel of the ukernel executor: one CTA per lane, each CTA drains its own
// CPU->device FIFO (uk_task.h) until it sees UK_EXIT.  Tasks of one lane run in order; lanes are
// independent and synchronise only through SIGNAL / WAIT counters in the symmetric heap, which is
// also how ranks talk to each other (a SIGNAL's target is usually the peer-mapped VA of the
// peer's counter).
//
// Reference role: experimental/ukernel/src/device/persistent_kernel_ops.cu:180,262 -- here the
// copy path is the same batched 16-byte ld/st engine the collectives use, reductions accumulate 16/8-bit floats in fp32, and completion is published twice:
// to pinned host memory (CPU polling) and to device memory (cuStreamWaitValue64 by user streams).
#include <stdio.h>

#include "../kernels/collectives_impl.cuh"
#include "../kernels/launch.h"
#include "uk_task.h"

namespace ub {

static __device__ __noinline__ void uk_abort(const UkWorkerArgs& w, int lane, uint64_t seq, const UkTask& t) {
  printf("[uccl_b200 ukernel] lane %d task %llu: WAIT timeout (addr %p want >= %llu)\n", lane,
         (unsigned long long)seq, (void*)t.sig_addr, (unsigned long long)t.sig_val);
  if (w.err) *w.err = 0x80000000u | 40u;
  __threadfence_system();
  __trap();
}

template <typename T, int OP>
__device__ __forceinline__ void uk_reduce_typed(char* dst, const char* a, const char* b, uint64_t bytes) {
  const bool aligned = ((((uintptr_t)dst | (uintptr_t)a | (uintptr_t)b) & 15) == 0);
  const uint64_t units = aligned ? bytes / 16 : 0;
  constexpr int U = 4;
  for (uint64_t u0 = threadIdx.x; u0 < units; u0 += (uint64_t)U * blockDim.x) {
    uint4 va[U], vb[U];
#pragma unroll
    for (int j = 0; j < U; ++j) {
      const uint64_t u = u0 + (uint64_t)j * blockDim.x;
      if (u < units) {
        va[j] = ld_v4(a + u * 16);
        vb[j] = ld_v4(b + u * 16);
      }
    }
#pragma unroll
    for (int j = 0; j < U; ++j) {
      const uint64_t u = u0 + (uint64_t)j * blockDim.x;
      if (u < units) {
        Vec16<T, OP> acc;
        acc.init(va[j]);
        acc.accum(vb[j]);
        st_v4(dst + u * 16, acc.pack_same());
      }
    }
  }
  // element tail (or everything, for unaligned operands)
  using A = typename AccOf<T>::type;
  const uint64_t first = units * 16 / sizeof(T), n = bytes / sizeof(T);
  for (uint64_t i = first + threadIdx.x; i < n; i += blockDim.x) {
    const A x = to_acc<A, T>(reinterpret_cast<const T*>(a)[i]);
    const A y = to_acc<A, T>(reinterpret_cast<const T*>(b)[i]);
    reinterpret_cast<T*>(dst)[i] = from_acc<T, A>(red_apply<OP, A>(x, y));
  }
}

template <typename T>
__device__ __forceinline__ void uk_reduce_ops(int op, char* dst, const char* a, const char* b, uint64_t bytes) {
  switch (op) {
    case kProd: uk_reduce_typed<T, kProd>(dst, a, b, bytes); break;
    case kMax: uk_reduce_typed<T, kMax>(dst, a, b, bytes); break;
    case kMin: uk_reduce_typed<T, kMin>(dst, a, b, bytes); break;
    default: uk_reduce_typed<T, kSum>(dst, a, b, bytes); break;
  }
}

__device__ __noinline__ void uk_reduce(const UkTask& t) {
  char* dst = reinterpret_cast<char*>(t.dst);
  const char* a = reinterpret_cast<const char*>(t.src);
  const char* b = reinterpret_cast<const char*>(t.src2);
  switch (t.dtype) {
    case kF32: uk_reduce_ops<float>(t.redop, dst, a, b, t.bytes); break;
    case kBF16: uk_reduce_ops<__nv_bfloat16>(t.redop, dst, a, b, t.bytes); break;
    case kF16: uk_reduce_ops<__half>(t.redop, dst, a, b, t.bytes); break;
    case kF64: uk_reduce_ops<double>(t.redop, dst, a, b, t.bytes); break;
    case kI8: uk_reduce_ops<int8_t>(t.redop, dst, a, b, t.bytes); break;
    case kU8: uk_reduce_ops<uint8_t>(t.redop, dst, a, b, t.bytes); break;
    case kI32: uk_reduce_ops<int32_t>(t.redop, dst, a, b, t.bytes); break;
    case kU32: uk_reduce_ops<uint32_t>(t.redop, dst, a, b, t.bytes); break;
    case kI64: uk_reduce_ops<int64_t>(t.redop, dst, a, b, t.bytes); break;
    case kU64: uk_reduce_ops<uint64_t>(t.redop, dst, a, b, t.bytes); break;
    case kF8E4M3: uk_reduce_ops<__nv_fp8_e4m3>(t.redop, dst, a, b, t.bytes); break;
    case kF8E5M2: uk_reduce_ops<__nv_fp8_e5m2>(t.redop, dst, a, b, t.bytes); break;
    default: break;
  }
}

__global__ void __launch_bounds__(512, 1) uk_worker_kernel(const __grid_constant__ UkWorkerArgs w) {
  const int lane = blockIdx.x;
  if (lane >= w.nlanes) return;
  const UkLane L = w.lane[lane];
  __shared__ UkTask s_task;
  __shared__ int s_quit;
  if (threadIdx.x == 0) s_quit = 0;
  bool voted = false;  // thread 0 only
  for (uint64_t seq = L.start;; ++seq) {
    if (threadIdx.x == 0) {
      const UkTask* slot = L.ring + (seq & (kUkRingEntries - 1));
      // the producer writes the 56 payload bytes, then releases `seq`; poll it with a
      // system-scope acquire so the payload read below cannot be satisfied early
      uint64_t idle_t0 = 0;
      uint32_t spins = 0;
      bool quit = false;
      while (true) {
        if (ld_acquire_sys(&slot->seq) == seq + 1) {
          if (voted) {  // withdraw the vote unless the exit is already committed
            unsigned int old = atomicAdd(w.votes, 0u);
            while (true) {
              if (old & kUkExitBit) {
                quit = true;  // the task stays in the ring for the next launch
                break;
              }
              const unsigned int prev = atomicCAS(w.votes, old, old - 1);
              if (prev == old) {
                voted = false;
                break;
              }
              old = prev;
            }
          }
          break;
        }
        if (w.idle_ns && ((++spins) & 0x3f) == 0) {
          const unsigned int v = atomicAdd(w.votes, 0u);
          if (v & kUkExitBit) {
            quit = true;
            break;
          }
          const uint64_t now = globaltimer_ns();
          if (idle_t0 == 0) idle_t0 = now;
          if (!voted && now - idle_t0 > w.idle_ns) {
            atomicAdd(w.votes, 1u);
            voted = true;
          }
          if (voted && (v & 0xffffu) == (unsigned int)w.nlanes) atomicCAS(w.votes, (unsigned int)w.nlanes, kUkExitBit | (unsigned int)w.nlanes);
        }
        __nanosleep(64);
      }
      if (quit) {
        s_quit = 1;
      } else {
        const uint4* p = reinterpret_cast<const uint4*>(slot);
        uint4* q = reinterpret_cast<uint4*>(&s_task);
#pragma unroll
        for (int i = 0; i < 4; ++i) q[i] = ld_volatile_v4(p + i);
      }
    }
    __syncthreads();
    if (s_quit) return;
    const uint32_t op = s_task.op;
    if (op == UK_COPY) {
      const uint64_t units = (s_task.bytes + 15) / 16;
      copy_bytes16(reinterpret_cast<char*>(s_task.dst), reinterpret_cast<const char*>(s_task.src), 0, units,
                   s_task.bytes, s_task.bytes);
    } else if (op == UK_REDUCE) {
      uk_reduce(s_task);
    } else if (op == UK_WAIT) {
      if (threadIdx.x == 0) {
        SpinGuard g(w.timeout_ns);
        const uint64_t* p = reinterpret_cast<const uint64_t*>(s_task.sig_addr);
        while (ld_acquire_sys(p) < s_task.sig_val) {
          if (g.expired()) uk_abort(w, lane, seq, s_task);
        }
      }
    }
    __syncthreads();  // every thread's stores of this task are issued
    if (threadIdx.x == 0) {
      if (op == UK_SIGNAL) {
        // the barrier above ordered the CTA's earlier stores before this thread; the fence + release
        // make them visible system-wide before the counter moves
        fence_acq_rel_sys();
        asm volatile("red.release.sys.global.add.u64 [%0], %1;" ::"l"(s_task.sig_addr), "l"(s_task.sig_val) : "memory");
      }
      __threadfence_system();
      *reinterpret_cast<volatile uint64_t*>(L.done_dev) = seq + 1;
      st_release_sys(L.done_host, seq + 1);
    }
    if (op == UK_EXIT) return;
    __syncthreads();  // s_task may be overwritten
  }
}

cudaError_t launch_uk_worker(const UkWorkerArgs& w, cudaStream_t st) {
  UB_LAUNCH((uk_worker_kernel), w.nlanes > 0 ? w.nlanes : 1, 512, 0, st, w);
  return cudaGetLastError();
}

}  // namespace ub
